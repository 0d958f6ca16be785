// fg_ftoa.cuh — f64 -> text exactly as Rust's `Display for f64` prints it (`value.to_string()`), the spelling of
// Record.ts and of F64 values in the reference's LTSV encoder (ltsv_encoder.rs:104-105, 114).
//
// Display takes the SHORTEST digit string that reads back to the same double, the closest one to the value when there
// are several (core::num::flt2dec::strategy::{grisu,dragon}::format_shortest), and lays it out positionally, never
// with an exponent and without a trailing ".0": 1, 1000000000000000000000 (1e21), 0.0000001 (1e-7), and for f64::MAX
// 17976931348623157 followed by 292 zeros; -0, NaN, inf, -inf.  (The GELF encoder's fg_dtoa.cuh is serde_json's Grisu2,
// which is not always shortest: the two must not be mixed up.)
//
// The digits come from Schubfach (Giulietti 2020, as in OpenJDK's DoubleToDecimal) with the 126-bit powers of ten of
// fg_ftoa_table.inc: exact, no fallback path.  Two departures from the Java code, both because Java prints at least two
// digits and Rust does not: the one-digit-shorter candidate is tried from s >= 10 on (Java: s >= 100), and the
// smallest subnormals are not scaled by 10 first.  Ties between two shortest candidates cannot occur for doubles, so
// the rounding of a tie (Java: even digit) never matters.
//
// The text can be 330 bytes long, so it is not formatted into a buffer: FtoaText holds the sign and digits (with the
// point where it falls inside them) and one run of zeros at a position, which the byte loop emits itself.
#pragma once
#include <stdint.h>

#include "fg_simt.cuh"

#ifdef FG_HOST_EMU
#define FG_FTOA_CONST const
#else
#define FG_FTOA_CONST __device__ const
#endif

namespace fg {

#include "fg_ftoa_table.inc"

// v = f * 10^e, f without trailing zeros (f > 0)
struct FtoaDec {
    uint64_t f;
    int e;
};

FG_DEV int ftoa_flog10pow2(int q) { return (int)(((long long)q * 661971961083ll) >> 41); }
FG_DEV int ftoa_flog10_three_quarters_pow2(int q) { return (int)(((long long)q * 661971961083ll - 274743187321ll) >> 41); }
FG_DEV int ftoa_flog2pow10(int k) { return (int)(((long long)k * 913124641741ll) >> 38); }

// the product g * cp rounded to odd (its high bits, with bit 0 set when any lower bit is)
FG_DEV uint64_t ftoa_rop(uint64_t g1, uint64_t g0, uint64_t cp) {
    const uint64_t x1 = __umul64hi(g0, cp);
    const uint64_t y0 = g1 * cp, y1 = __umul64hi(g1, cp);
    const uint64_t z = (y0 >> 1) + x1;
    const uint64_t vbp = y1 + (z >> 63);
    return vbp | (((z & 0x7FFFFFFFFFFFFFFFull) + 0x7FFFFFFFFFFFFFFFull) >> 63);
}

FG_DEV FtoaDec ftoa_strip(uint64_t f, int e) {
    while (f % 10u == 0u) {
        f /= 10u;
        ++e;
    }
    return FtoaDec{f, e};
}

// shortest closest decimal of c * 2^q (c > 0)
FG_DEV FtoaDec ftoa_to_decimal(int q, uint64_t c, bool normal_lowest) {
    const uint64_t out = c & 1u;
    const uint64_t cb = c << 2, cbr = cb + 2;
    uint64_t cbl;
    int k;
    if (!normal_lowest) {
        cbl = cb - 2;
        k = ftoa_flog10pow2(q);
    } else {  // c = 2^52 of a normal binade: the gap below is half the gap above
        cbl = cb - 1;
        k = ftoa_flog10_three_quarters_pow2(q);
    }
    const int h = q + ftoa_flog2pow10(-k) + 2;
    const uint64_t g1 = kFtoaG[2 * (k + 324)], g0 = kFtoaG[2 * (k + 324) + 1];
    const uint64_t vb = ftoa_rop(g1, g0, cb << h), vbl = ftoa_rop(g1, g0, cbl << h), vbr = ftoa_rop(g1, g0, cbr << h);
    const uint64_t s = vb >> 2;
    if (s >= 10u) {  // one digit fewer: the one multiple of 10 the interval may hold
        const uint64_t sp10 = 10u * __umul64hi(s, 1844674407370955168ull), tp10 = sp10 + 10u;
        const bool upin = vbl + out <= sp10 << 2, wpin = (tp10 << 2) + out <= vbr;
        if (upin != wpin) return ftoa_strip(upin ? sp10 : tp10, k);
    }
    const uint64_t t = s + 1u;
    const bool uin = vbl + out <= s << 2, win = (t << 2) + out <= vbr;
    if (uin != win) return ftoa_strip(uin ? s : t, k);
    const long long cmp = (long long)(vb - ((s + t) << 1));
    return ftoa_strip(cmp < 0 || (cmp == 0 && (s & 1u) == 0u) ? s : t, k);
}

// |v| for finite nonzero v
FG_DEV FtoaDec ftoa_shortest(uint64_t bits) {
    const uint64_t t = bits & 0x000FFFFFFFFFFFFFull;
    const int bq = (int)((bits >> 52) & 0x7FFu);
    if (bq == 0) return ftoa_to_decimal(-1074, t, false);  // subnormal
    const int mq = 1075 - bq;
    const uint64_t c = t | (1ull << 52);
    if (0 < mq && mq < 53) {  // an integer below 2^53: exact
        const uint64_t f = c >> mq;
        if (f << mq == c) return ftoa_strip(f, 0);
    }
    return ftoa_to_decimal(-mq, c, t == 0u && bq > 1);
}

// A number's text: buf[0, zpos), then zlen '0' bytes, then buf[zpos, blen).  Total length blen + zlen (<= 24 + 308).
struct FtoaText {
    uint8_t buf[24];
    int blen, zpos, zlen;
    __device__ __forceinline__ uint8_t at(int k) const { return k < zpos ? buf[k] : (k < zpos + zlen ? (uint8_t)'0' : buf[k - zlen]); }
    __device__ __forceinline__ int len() const { return blen + zlen; }
};

FG_DEV int ftoa_digits(uint64_t f, uint8_t* out) {  // decimal digits of f, returns their count
    int d = 1;
    for (uint64_t x = f; x >= 10u; x /= 10u) ++d;
    for (int k = d - 1; k >= 0; --k, f /= 10u) out[k] = (uint8_t)('0' + (uint32_t)(f % 10u));
    return d;
}

FG_DEV void ftoa_word(FtoaText& t, uint32_t w, int n) {  // n <= 4 bytes of w, low byte first
    for (int k = 0; k < n; ++k) t.buf[k] = (uint8_t)(w >> (8 * k));
    t.blen = n;
    t.zpos = n;
    t.zlen = 0;
}

// Display for f64
FG_DEV void f64_display(double v, FtoaText& t) {
    const uint64_t bits = (uint64_t)__double_as_longlong(v);
    const bool neg = (bits >> 63) != 0u;
    const uint64_t mag = bits & 0x7FFFFFFFFFFFFFFFull;
    if (mag >= 0x7FF0000000000000ull) {
        if (mag > 0x7FF0000000000000ull) ftoa_word(t, 0x4E614Eu, 3);                // "NaN"
        else if (neg) ftoa_word(t, 0x666E692Du, 4);                                  // "-inf"
        else ftoa_word(t, 0x666E69u, 3);                                             // "inf"
        return;
    }
    if (mag == 0u) {
        if (neg) ftoa_word(t, 0x302Du, 2);  // "-0"
        else ftoa_word(t, 0x30u, 1);
        return;
    }
    const FtoaDec d = ftoa_shortest(mag);
    int n = 0;
    if (neg) t.buf[n++] = '-';
    uint8_t dig[20];
    const int nd = ftoa_digits(d.f, dig), point = nd + d.e;  // digits before the point
    t.zlen = 0;
    if (d.e >= 0) {  // ddd000
        for (int k = 0; k < nd; ++k) t.buf[n++] = dig[k];
        t.zpos = n;
        t.zlen = d.e;
    } else if (point > 0) {  // dd.ddd
        for (int k = 0; k < nd; ++k) {
            if (k == point) t.buf[n++] = '.';
            t.buf[n++] = dig[k];
        }
        t.zpos = n;
    } else {  // 0.000ddd
        t.buf[n++] = '0';
        t.buf[n++] = '.';
        t.zpos = n;
        t.zlen = -point;
        for (int k = 0; k < nd; ++k) t.buf[n++] = dig[k];
    }
    t.blen = n;
}

// I64 / U64 (and the u8 fields of a Record) in decimal
FG_DEV void int_display(uint64_t v, bool is_signed, FtoaText& t) {
    int n = 0;
    if (is_signed && (long long)v < 0) {
        t.buf[n++] = '-';
        v = 0ull - v;  // i64::MIN too
    }
    n += ftoa_digits(v, t.buf + n);
    t.blen = t.zpos = n;
    t.zlen = 0;
}

}  // namespace fg
