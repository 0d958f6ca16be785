// fg_common.cuh — device helpers shared by the per-format line parsers.
//
// Everything here is integer/byte work except the two IEEE operations of the
// timestamp recipe (utils/mod.rs:24-28).  Never compile this with
// --use_fast_math: the f64 conversion and division must be round-to-nearest.
#pragma once
#include <stdint.h>

#include "fg_simt.cuh"

namespace fg {

typedef const uint8_t* __restrict__ bytes_t;

FG_DEV bool is_digit(uint32_t c) { return (c - (uint32_t)'0') <= 9u; }

// what the splitter leaves of record [lo, hi): mode 1 = BufRead::lines (line_splitter.rs:17: the '\n' goes, and one '\r'
// before it), 2 = BufRead::split(0) (nul_splitter.rs:18: only the NUL goes), 0 = the caller framed the record; returns
// the new hi.  A record that is not UTF-8 is reported and skipped (:22-25): that flag is the call site's to look up.
FG_DEV int strip_terminator(bytes_t p, int lo, int hi, int mode) {
    if (mode == 0 || hi <= lo) return hi;
    if (mode == 2) return p[hi - 1] == 0 ? hi - 1 : hi;
    if (p[hi - 1] == '\n') {
        --hi;
        if (hi > lo && p[hi - 1] == '\r') --hi;
    }
    return hi;
}

// A CTA stages the byte span of its lines with one bulk copy of 16-byte granules (fg_tma.cuh): the span starts at the
// granule that holds the first line's first byte and is copied up to the end of the granule that holds its last byte
// (<= tile_bytes, a multiple of 512, when the lines fit; the input buffer is padded).
FG_DEV int span_base(int first_offset) { return first_offset & ~15; }
FG_DEV uint32_t span_copy_bytes(int base, int oend) { return (uint32_t)((oend - base) + 15) & ~15u; }

// ---------------------------------------------------------------------------
// str::trim / trim_end — Unicode White_Space, matched byte-wise on valid UTF-8
// (rfc5424_decoder.rs:46,167).  U+0009-000D, 0020, 0085, 00A0, 1680,
// 2000-200A, 2028, 2029, 202F, 205F, 3000.
// ---------------------------------------------------------------------------
FG_DEV bool is_ascii_ws(uint32_t c) { return (c - 9u) <= 4u || c == 32u; }

// length of the whitespace char ending at hi (exclusive) within [lo,hi); 0 if none
FG_DEV int ws_len_back(bytes_t p, int lo, int hi) {
    uint32_t l = p[hi - 1];
    if (l < 0x80u) return is_ascii_ws(l) ? 1 : 0;
    if (hi - lo < 2) return 0;
    uint32_t m = p[hi - 2];
    if (m == 0xC2u) return (l == 0x85u || l == 0xA0u) ? 2 : 0;
    if (hi - lo < 3) return 0;
    uint32_t f = p[hi - 3];
    if (f == 0xE2u) {
        if (m == 0x80u) return ((l >= 0x80u && l <= 0x8Au) || l == 0xA8u || l == 0xA9u || l == 0xAFu) ? 3 : 0;
        return (m == 0x81u && l == 0x9Fu) ? 3 : 0;
    }
    if (f == 0xE1u) return (m == 0x9Au && l == 0x80u) ? 3 : 0;
    if (f == 0xE3u) return (m == 0x80u && l == 0x80u) ? 3 : 0;
    return 0;
}
FG_DEV int ws_len_front(bytes_t p, int lo, int hi) {
    uint32_t c0 = p[lo];
    if (c0 < 0x80u) return is_ascii_ws(c0) ? 1 : 0;
    if (hi - lo < 2) return 0;
    uint32_t c1 = p[lo + 1];
    if (c0 == 0xC2u) return (c1 == 0x85u || c1 == 0xA0u) ? 2 : 0;
    if (hi - lo < 3) return 0;
    uint32_t c2 = p[lo + 2];
    if (c0 == 0xE2u) {
        if (c1 == 0x80u) return ((c2 >= 0x80u && c2 <= 0x8Au) || c2 == 0xA8u || c2 == 0xA9u || c2 == 0xAFu) ? 3 : 0;
        return (c1 == 0x81u && c2 == 0x9Fu) ? 3 : 0;
    }
    if (c0 == 0xE1u) return (c1 == 0x9Au && c2 == 0x80u) ? 3 : 0;
    if (c0 == 0xE3u) return (c1 == 0x80u && c2 == 0x80u) ? 3 : 0;
    return 0;
}
FG_DEV int trim_end(bytes_t p, int lo, int hi) {
    while (hi > lo) {
        int w = ws_len_back(p, lo, hi);
        if (!w) break;
        hi -= w;
    }
    return hi;
}
FG_DEV int trim_start(bytes_t p, int lo, int hi) {
    while (lo < hi) {
        int w = ws_len_front(p, lo, hi);
        if (!w) break;
        lo += w;
    }
    return lo;
}

// ---------------------------------------------------------------------------
// Rust integer from_str (SURVEY.md Appendix B)
// ---------------------------------------------------------------------------
// u8::from_str over [a,b): [+]digit+, value <= 255
FG_DEV bool parse_u8(bytes_t p, int a, int b, uint32_t& out) {
    if (a >= b) return false;
    if (p[a] == '+') ++a;
    if (a >= b) return false;
    uint32_t v = 0;
    for (; a < b; ++a) {
        uint32_t d = (uint32_t)p[a] - '0';
        if (d > 9u) return false;
        v = v * 10u + d;
        if (v > 255u) return false;
    }
    out = v;
    return true;
}
FG_DEV bool parse_u64(bytes_t p, int a, int b, uint64_t& out) {
    if (a >= b) return false;
    if (p[a] == '+') ++a;
    if (a >= b) return false;
    uint64_t v = 0;
    for (; a < b; ++a) {
        uint32_t d = (uint32_t)p[a] - '0';
        if (d > 9u) return false;
        if (v > (0xFFFFFFFFFFFFFFFFull - d) / 10ull) return false;
        v = v * 10ull + d;
    }
    out = v;
    return true;
}
FG_DEV bool parse_i64(bytes_t p, int a, int b, int64_t& out) {
    if (a >= b) return false;
    bool neg = false;
    if (p[a] == '+') ++a;
    else if (p[a] == '-') { neg = true; ++a; }
    if (a >= b) return false;
    uint64_t lim = neg ? (1ull << 63) : 0x7FFFFFFFFFFFFFFFull;
    uint64_t v = 0;
    for (; a < b; ++a) {
        uint32_t d = (uint32_t)p[a] - '0';
        if (d > 9u) return false;
        if (v > (lim - d) / 10ull) return false;
        v = v * 10ull + d;
    }
    out = neg ? (int64_t)(0ull - v) : (int64_t)v;
    return true;
}

// ---------------------------------------------------------------------------
// `time` 0.3 calendar + the reference timestamp recipe
// ---------------------------------------------------------------------------
FG_DEV bool is_leap(int y) { return ((y & 3) == 0 && (y % 100) != 0) || (y % 400) == 0; }
FG_DEV int days_in_month(int y, int m) {
    // 31 28 31 30 31 30 31 31 30 31 30 31 packed 2 bits (value-28) per month
    int d = 28 + ((0xEEFBB3 >> ((m - 1) * 2)) & 3);
    return (m == 2 && is_leap(y)) ? 29 : d;
}
// proleptic Gregorian days since 1970-01-01 (y in [-9999, 9999])
FG_DEV int days_from_civil(int y, int m, int d) {
    y -= m <= 2;
    int era = (y >= 0 ? y : y - 399) / 400;
    int yoe = y - era * 400;
    int doy = (153 * (m + (m > 2 ? -3 : 9)) + 2) / 5 + d - 1;
    int doe = yoe * 365 + yoe / 4 - yoe / 100 + doy;
    return era * 146097 + doe - 719468;
}

// (sign, 128-bit magnitude) -> f64 with ONE round-to-nearest-even, i.e. Rust's
// `i128 as f64` (utils/mod.rs:26).
FG_DEV double i128_to_f64(bool neg, uint64_t hi, uint64_t lo) {
    double d;
    if (hi == 0) {
        d = __ull2double_rn(lo);
    } else {
        int sh = __clzll((long long)hi);  // hi != 0 -> 0..63
        uint64_t top = sh ? ((hi << sh) | (lo >> (64 - sh))) : hi;
        uint64_t rest = sh ? (lo << sh) : lo;
        top |= (rest != 0) ? 1ull : 0ull;  // sticky bit: only influences the tie break
        d = __ull2double_rn(top);
        // exact scaling by 2^(64-sh)
        d = __dmul_rn(d, __hiloint2double((1023 + 64 - sh) << 20, 0));
    }
    return neg ? -d : d;
}

// seconds since epoch (may be negative) + nanos in [0,1e9) -> ts
// = fl(fl(nanos_i128) / 1e9)   (two IEEE roundings, like the reference)
FG_DEV double unix_nanos_to_ts(int64_t secs, uint32_t ns) {
    bool neg = secs < 0;
    uint64_t hi, lo;
    if (!neg) {
        uint64_t s = (uint64_t)secs;
        lo = s * 1000000000ull;
        hi = __umul64hi(s, 1000000000ull);
        uint64_t l2 = lo + ns;
        hi += (l2 < lo);
        lo = l2;
    } else {
        uint64_t s = (uint64_t)(-secs);  // |secs| >= 1 so the magnitude stays positive
        lo = s * 1000000000ull;
        hi = __umul64hi(s, 1000000000ull);
        uint64_t l2 = lo - ns;
        hi -= (l2 > lo);
        lo = l2;
    }
    return __ddiv_rn(i128_to_f64(neg, hi, lo), 1e9);
}

struct DateTime {
    int year, month, day, hour, minute, second;
    uint32_t nanos;
    int offset_seconds;
};

// Date::from_calendar_date + Time::from_hms_nano + assume_offset + (optional)
// is_valid_leap_second_stand_in, then the reference's f64 recipe.
FG_DEV bool finish_datetime(const DateTime& t, bool leap_in, double& ts) {
    if (t.month < 1 || t.month > 12) return false;
    if (t.day < 1 || t.day > days_in_month(t.year, t.month)) return false;
    if (t.hour > 23 || t.minute > 59 || t.second > 59) return false;
    int64_t local = (int64_t)days_from_civil(t.year, t.month, t.day) * 86400 + t.hour * 3600 + t.minute * 60 + t.second;
    int64_t utc = local - t.offset_seconds;
    if (leap_in) {
        if (t.nanos != 999999999u) return false;
        int64_t days = utc >= 0 ? utc / 86400 : -((-utc + 86399) / 86400);
        int64_t sod = utc - days * 86400;
        if (sod != 86399) return false;
        int64_t z = days + 719468;
        int64_t era = (z >= 0 ? z : z - 146096) / 146097;
        int doe = (int)(z - era * 146097);
        int yoe = (doe - doe / 1460 + doe / 36524 - doe / 146096) / 365;
        int y = yoe + (int)era * 400;
        int doy = doe - (365 * yoe + yoe / 4 - yoe / 100);
        int mp = (5 * doy + 2) / 153;
        int d = doy - (153 * mp + 2) / 5 + 1;
        int m = mp < 10 ? mp + 3 : mp - 9;
        y += m <= 2;
        if (d != days_in_month(y, m)) return false;
    }
    ts = unix_nanos_to_ts(utc, t.nanos);
    return true;
}

FG_DEV bool two_digits(bytes_t p, int& i, int b, int& out) {
    if (i + 2 > b) return false;
    uint32_t x = (uint32_t)p[i] - '0', y = (uint32_t)p[i + 1] - '0';
    if (x > 9u || y > 9u) return false;
    out = (int)(x * 10u + y);
    i += 2;
    return true;
}
FG_DEV bool four_digits(bytes_t p, int& i, int b, int& out) {
    if (i + 4 > b) return false;
    uint32_t v = 0;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        uint32_t d = (uint32_t)p[i + k] - '0';
        if (d > 9u) return false;
        v = v * 10u + d;
    }
    out = (int)v;
    i += 4;
    return true;
}
// any_digit+ ; digits after the 9th are consumed and dropped (time's subsecond rule)
FG_DEV bool subsecond(bytes_t p, int& i, int b, uint32_t& nanos) {
    if (i >= b || !is_digit(p[i])) return false;
    uint32_t v = 0, mult = 100000000u;
    while (i < b) {
        uint32_t d = (uint32_t)p[i] - '0';
        if (d > 9u) break;
        v += d * mult;
        mult /= 10u;
        ++i;
    }
    nanos = v;
    return true;
}

// OffsetDateTime::parse(s, &Rfc3339) over [a,b)  (rfc5424_decoder.rs:94-99, ltsv_decoder.rs:224-229)
FG_DEV bool parse_rfc3339(bytes_t p, int a, int b, double& ts) {
    int i = a;
    DateTime t;
    t.nanos = 0;
    if (!four_digits(p, i, b, t.year)) return false;
    if (i >= b || p[i] != '-') return false;
    ++i;
    if (!two_digits(p, i, b, t.month)) return false;
    if (i >= b || p[i] != '-') return false;
    ++i;
    if (!two_digits(p, i, b, t.day)) return false;
    if (i >= b || (p[i] | 0x20u) != 't') return false;
    ++i;
    if (!two_digits(p, i, b, t.hour)) return false;
    if (i >= b || p[i] != ':') return false;
    ++i;
    if (!two_digits(p, i, b, t.minute)) return false;
    if (i >= b || p[i] != ':') return false;
    ++i;
    if (!two_digits(p, i, b, t.second)) return false;
    if (i < b && p[i] == '.') {
        ++i;
        if (!subsecond(p, i, b, t.nanos)) return false;
    }
    if (i >= b) return false;
    uint32_t c = p[i];
    if ((c | 0x20u) == 'z') {
        ++i;
        t.offset_seconds = 0;
    } else {
        if (c != '+' && c != '-') return false;
        ++i;
        int oh, om;
        if (!two_digits(p, i, b, oh)) return false;
        if (i >= b || p[i] != ':') return false;
        ++i;
        if (!two_digits(p, i, b, om)) return false;
        if (oh > 25 || om > 59) return false;  // UtcOffset::from_hms range
        int off = oh * 3600 + om * 60;
        t.offset_seconds = (c == '-') ? -off : off;
    }
    if (i != b) return false;  // UnexpectedTrailingCharacters
    bool leap = false;
    if (t.second == 60) {
        t.second = 59;
        t.nanos = 999999999u;
        leap = true;
    }
    return finish_datetime(t, leap, ts);
}

#ifndef FG_HOST_EMU
// ---------------------------------------------------------------------------
// small CTA-wide exclusive scan (blockDim.x <= 1024) used to place each line's
// structured-data entries in the side table
// ---------------------------------------------------------------------------
FG_DEV uint32_t block_exclusive_scan(uint32_t v, uint32_t* warp_sums /* [32] smem */, uint32_t& total) {
    const uint32_t lane = threadIdx.x & 31u, wid = threadIdx.x >> 5;
    uint32_t x = v;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
        uint32_t y = __shfl_up_sync(0xFFFFFFFFu, x, d);
        if (lane >= (uint32_t)d) x += y;
    }
    if (lane == 31u) warp_sums[wid] = x;
    __syncthreads();
    const uint32_t nw = (blockDim.x + 31u) >> 5;
    if (wid == 0) {
        uint32_t w = lane < nw ? warp_sums[lane] : 0u;
        uint32_t s = w;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
            uint32_t y = __shfl_up_sync(0xFFFFFFFFu, s, d);
            if (lane >= (uint32_t)d) s += y;
        }
        warp_sums[lane] = s - w;  // exclusive prefix of warp totals
        if (lane == 31u) warp_sums[32] = s;
    }
    __syncthreads();
    total = warp_sums[32];
    uint32_t r = warp_sums[wid] + x - v;
    return r;
}
#endif  // FG_HOST_EMU

}  // namespace fg
