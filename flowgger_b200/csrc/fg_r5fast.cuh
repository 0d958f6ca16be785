// fg_r5fast.cuh — RFC5424 fast path: structural bitmaps + one-pair-per-step walk over a shared-memory tile.
//
// H100-native replacement for RFC5424Decoder::decode
// (flowgger src/flowgger/decoder/rfc5424_decoder.rs:18-49) and its helpers BOM::parse :63-71,
// parse_pri_version :74-92, rfc3339_to_unix :94-99, parse_data :127-161, parse_msg :163-172,
// parse_sd_data :174-242 — for REGULAR lines, i.e. lines of the shape every syslog sender emits:
//     <PRI>1 TS HOST APP PROCID MSGID (-|[id name="value" name="value"][id ...]) MSG
// The walker proves regularity as it goes; the first byte that does not fit (a BOM, a header field holding a
// delimiter-class byte, a lower-case 't', a stray quote, two spaces between params, any malformed line ...) hands the
// line to the exact scanner of the slow kernel (fg_rfc5424.cuh), which restates the reference's state machine arm by
// arm and produces every error string.  Regular lines therefore never carry an error status.
//
//   stage 1  r5_classify16: every thread takes 16-byte granules of the flat tile (LDS.128, conflict-free, all 32 lanes
//            busy) and writes one bit per byte into a bitmap (exact per byte, no cross-byte carries):
//              I  "may end a token", a cheap SUPERSET of the delimiters (7 SWAR ops per 4 bytes):
//                   b <= 0x22            control bytes, ' ', '!', '"'
//                   (b & 0x1E) == 0x1C   0x1C 0x1D '<' '=' '\\' ']' '|' '}'
//                   b >= 0x7F            DEL and every non-ASCII byte
//                 every byte that is NOT flagged is a legal SD-NAME character (:188-192) and is neither a space, a
//                 quote, '=', ']' nor a backslash.
//   stage 2  r5_regular: one thread per line.  Header: the first six flagged bytes must be the six spaces of
//            splitn(7, ' ') (:23).  PRI and the RFC3339 stamp are parsed at fixed offsets.  Structured data: ONE
//            name="value" pair per loop iteration — a find-first-set on I gives the '=' that ends the name, the flagged
//            bytes after the opening quote lead to the closing one — and the 32 lines of a warp advance in lock step, so a
//            warp pays the maximum number of PAIRS over its lanes.
//
// Structured-data rows are staged as 8-byte packed entries (u16 positions relative to the line start) in the line's OWN
// already-consumed bytes of the tile: slot k may be written once the cursor has passed its last byte.
//
// The unescape of SD values (:105-125) is done by post5424_kernel (fg_parse5424.cu: unescape_lines) into the batch's arena; this
// walker only marks the pairs whose value holds a backslash.
#pragma once
#include "fg_common.cuh"
#include "fg_status.h"

namespace fg {

// ---- stage 1 ----------------------------------------------------------------------------------------------------
// 0x80 in every byte of w that is "interesting" (see the header comment); exact per byte.
FG_DEV uint32_t r5_flags(uint32_t w) {
    const uint32_t low = w & 0x7F7F7F7Fu;
    const uint32_t a2 = low + 0x5D5D5D5Du;                    // bit 7: low >= 0x23   (max 0xDC: no carry out of the byte)
    const uint32_t a1 = low + 0x01010101u;                    // bit 7: low == 0x7F
    const uint32_t x = (w & 0x1E1E1E1Eu) ^ 0x1C1C1C1Cu;       // 0 iff (b & 0x1E) == 0x1C
    const uint32_t a3 = x + 0x7F7F7F7Fu;                      // bit 7: x != 0        (x <= 0x1E: no carry)
    return (~a2 | a1 | w | ~a3) & 0x80808080u;
}
// the four 0x80 flags of a word -> bits 28..31 (byte j -> bit 28 + j); bits 24..27 of the product are always 0
FG_DEV uint32_t r5_nibble_top(uint32_t f) { return f * 0x00204081u; }
FG_DEV uint32_t r5_gather16(uint32_t f0, uint32_t f1, uint32_t f2, uint32_t f3) {
    const uint32_t n0 = r5_nibble_top(f0), n1 = r5_nibble_top(f1), n2 = r5_nibble_top(f2), n3 = r5_nibble_top(f3);
    return (n0 >> 28) | ((n1 >> 24) & 0xF0u) | ((n2 >> 20) & 0xF00u) | ((n3 >> 16) & 0xF000u);
}
FG_DEV uint32_t r5_classify16(uint32_t w0, uint32_t w1, uint32_t w2, uint32_t w3) {
    return r5_gather16(r5_flags(w0), r5_flags(w1), r5_flags(w2), r5_flags(w3));
}
// ---- stage 2 ----------------------------------------------------------------------------------------------------
// 32 bitmap bits starting at tile position t (bit 0 = byte t).  bm needs one readable word past the last granule.
FG_DEV uint32_t r5_window(const uint32_t* bm, int t) {
    const int k = t >> 5;
    return fg_funnel_r(bm[k], bm[k + 1], (uint32_t)t & 31u);
}

// packed 8-byte side-table rows (positions relative to the line start, < 65536); bits 63..62 select the kind
//   10 header: sd_id start | sd_id end << 16 | #pairs << 32
//   00 pair  : name_start | name_end << 16 | value_end << 32 | flags << 48   (value starts at name_end + 2)
//              flag bit 48 (kE8Esc) = the value holds a backslash; such rows only exist between parse5424_kernel and
//              post5424_kernel (unescape_lines), which rewrites them as
//   01 arena pair: name_start | name_end << 16 | (arena offset / 2) << 32; the arena record is [u16 length][bytes],
//              2-byte aligned: the value with unescape_sd_value (:105-125) already applied
constexpr unsigned long long kE8Esc = 1ull << 48;
constexpr unsigned long long kE8Header = 1ull << 63;
constexpr unsigned long long kE8Arena = 1ull << 62;
FG_DEV unsigned long long r5_pack_pair8(int ns, int ne, int ve, bool esc) {
    return (unsigned long long)(uint32_t)ns | ((unsigned long long)(uint32_t)ne << 16) | ((unsigned long long)(uint32_t)ve << 32) |
           (esc ? kE8Esc : 0ull);
}
FG_DEV unsigned long long r5_pack_header8(int es, int id_end, uint32_t pairs) {
    return (unsigned long long)(uint32_t)es | ((unsigned long long)(uint32_t)id_end << 16) | ((unsigned long long)(pairs & 0xFFFFu) << 32) | kE8Header;
}

struct R5Fast {
    double ts;
    uint32_t status, facility, severity, flags;
    int sp1, sp2, sp3, sp4, sp5;  // relative to the line start: hostname = [sp1+1, sp2), appname = [sp2+1, sp3), ...
    int msg_o, msg_l;             // msg span; msg_l == 0 => msg None and msg_o = end of full_msg
    uint32_t n_entries;           // 8-byte rows staged at stage[0 .. n_entries)
    unsigned long long* stage;
    bool esc;   // some value holds a backslash (the line goes on the unescape work list)
};

// unescape_sd_value (rfc5424_decoder.rs:105-125) over the raw value bytes v[0, len): `\"` `\\` `\]` drop the backslash,
// any other escaped byte keeps it, a trailing lone backslash is dropped.  Returns the unescaped length; writes when out != nullptr.
FG_DEV int r5_unescape(const uint8_t* v, int len, uint8_t* out) {
    int o = 0;
    bool esc = false;
    for (int k = 0; k < len; ++k) {
        const uint8_t c = v[k];
        if (!esc) {
            if (c == '\\') esc = true;
            else {
                if (out) out[o] = c;
                ++o;
            }
        } else {
            if (c != '"' && c != '\\' && c != ']') {
                if (out) out[o] = '\\';
                ++o;
            }
            if (out) out[o] = c;
            ++o;
            esc = false;
        }
    }
    return o;
}

// the same rewrite, write-only and one decision per raw byte pair (the hot loop of unescape_lines)
FG_DEV int r5_unescape_to(const uint8_t* v, int len, uint8_t* out) {
    int o = 0;
    for (int k = 0; k < len; ++k) {
        const uint32_t c = v[k];
        if (c != '\\') {
            out[o++] = (uint8_t)c;
        } else if (k + 1 < len) {  // a trailing lone backslash is dropped
            const uint32_t d = v[++k];
            if (d != '"' && d != '\\' && d != ']') out[o++] = '\\';
            out[o++] = (uint8_t)d;
        }
    }
    return o;
}

constexpr uint32_t kFlagWide = 0x80u;  // FG_FLAG_WIDE

// Days from 1970-01-01 of a date already known to be valid, and the calendar checks of the fast stamp parser
FG_DEV uint32_t r5_digit(const uint8_t* T, int at, uint32_t& worst) {
    const uint32_t d = (uint32_t)T[at] - (uint32_t)'0';
    worst = max(worst, d);  // every "digit" was one iff the maximum is <= 9
    return d;
}

// T: tile bytes (shared memory), bmI: its bitmap; the line is T[ls, le).  Idle lanes pass ls == le.
// Returns true when the line is regular and `r` holds its Record fields (status is always Ok); false hands the line to
// the slow kernel.  ALL lanes of a warp must call this together.
FG_DEV bool r5_regular(uint8_t* T, const uint32_t* bmI, int ls, int le, R5Fast& r) {
    r.ts = 0.0;
    r.status = FG_ST_OK;
    r.facility = 0xFFu;
    r.severity = 0xFFu;
    r.flags = 0;
    r.sp1 = r.sp2 = r.sp3 = r.sp4 = r.sp5 = 0;
    r.msg_o = r.msg_l = 0;
    r.n_entries = 0;
    r.stage = nullptr;
    r.esc = false;
    bool ok = le - ls >= 32;  // "<1>1 2015-08-05T15:53:45Z h a p m -" is 35 bytes: nothing shorter is a complete line

    // ---- splitn(7, ' ') :23 — the first six flagged bytes after the leading '<' must be the six spaces -------------
    int sp[6];
    {
        int t = ls + 1;  // the '<' that opens PRI is itself a flagged byte
#pragma unroll
        for (int k = 0; k < 6; ++k) {
            uint32_t W = r5_window(bmI, t);
            if (k == 1 && W == 0u) {  // the stamp may be longer than 31 bytes (nanoseconds + offset: 35): look once more
                t += 32;
                W = r5_window(bmI, t);
            }
            t += fg_ffs(W) - 1;  // W == 0: t - 1, caught by the check below
            ok = ok && W != 0u && t < le && T[t] == ' ';
            sp[k] = t;
            t = ok ? t + 1 : ls;
        }
    }
    // ---- parse_pri_version :74-92: '<' 1..3 digits '>' '1' -----------------------------------------------------
    uint32_t bad = 0;
    {
        const int l0 = sp[0] - ls;  // 4..6
        ok = ok && T[ls] == '<' && l0 >= 4 && l0 <= 6;
        const int gt = ok ? sp[0] - 2 : ls;
        ok = ok && T[gt] == '>' && T[gt + 1] == '1';
        uint32_t pri = 0;
        for (int q = ls + 1; q < gt; ++q) pri = pri * 10u + r5_digit(T, q, bad);  // 1..3 iterations
        ok = ok && pri <= 255u;
        r.facility = pri >> 3;
        r.severity = pri & 7u;
    }
    // ---- rfc3339_to_unix :94-99 at fixed offsets: YYYY-MM-DDTHH:MM:SS[.f{1,9}](Z|+HH:MM|-HH:MM) ---------------------
    {
        const int a = ok ? sp[0] + 1 : ls, e = ok ? sp[1] : ls;
        const int L = e - a;
        ok = ok && L >= 20;
        const int z = ok ? e - 1 : ls;         // 'Z', or the last digit of the offset
        const bool zulu = T[z] == 'Z';
        const int zone = zulu ? z : z - 5;     // where the zone designator starts
        DateTime t;
        t.year = (int)(r5_digit(T, a, bad) * 1000u + r5_digit(T, a + 1, bad) * 100u + r5_digit(T, a + 2, bad) * 10u + r5_digit(T, a + 3, bad));
        t.month = (int)(r5_digit(T, a + 5, bad) * 10u + r5_digit(T, a + 6, bad));
        t.day = (int)(r5_digit(T, a + 8, bad) * 10u + r5_digit(T, a + 9, bad));
        t.hour = (int)(r5_digit(T, a + 11, bad) * 10u + r5_digit(T, a + 12, bad));
        t.minute = (int)(r5_digit(T, a + 14, bad) * 10u + r5_digit(T, a + 15, bad));
        t.second = (int)(r5_digit(T, a + 17, bad) * 10u + r5_digit(T, a + 18, bad));
        ok = ok && T[a + 4] == '-' && T[a + 7] == '-' && T[a + 10] == 'T' && T[a + 13] == ':' && T[a + 16] == ':';
        // fraction: [a + 19, zone) is empty or '.' + 1..9 digits
        const int fl = zone - (a + 19);
        ok = ok && (fl == 0 || (fl >= 2 && fl <= 10 && T[a + 19] == '.'));
        uint32_t nanos = 0, mult = 100000000u;
#pragma unroll
        for (int k = 0; k < 9; ++k) {
            if (k + 1 < fl) nanos += r5_digit(T, a + 20 + k, bad) * mult;
            mult /= 10u;
        }
        t.nanos = nanos;
        int off = 0;
        if (!zulu) {
            const uint32_t sg = T[zone];
            const int oh = (int)(r5_digit(T, zone + 1, bad) * 10u + r5_digit(T, zone + 2, bad));
            const int om = (int)(r5_digit(T, zone + 4, bad) * 10u + r5_digit(T, zone + 5, bad));
            ok = ok && (sg == '+' || sg == '-') && T[zone + 3] == ':' && oh <= 23 && om <= 59 && zone >= a + 19;
            off = oh * 3600 + om * 60;
            if (sg == '-') off = -off;
        }
        t.offset_seconds = off;
        ok = ok && bad <= 9u && t.second <= 59;  // :60 (leap second stand-in) is the slow path's business
        if (!ok) { t.year = 2000; t.month = 1; t.day = 1; t.hour = t.minute = t.second = 0; t.nanos = 0; t.offset_seconds = 0; }
        double ts = 0.0;
        ok = finish_datetime(t, false, ts) && ok;
        r.ts = ts;
    }
    fg_syncwarp();

    // ---- parse_data :127-161 on part6 = [sp5+1, le) ------------------------------------------------
    const int d = ok ? sp[5] + 1 : ls;
    int msg_from = le;
    bool walk = false;
    ok = ok && d < le;
    if (ok) {
        const uint32_t c0 = T[d];
        if (c0 == '-') msg_from = d + 1;
        else if (c0 == '[') walk = true;
        else ok = false;
    }
    {
        // Structured data: one name="value" pair per iteration and lane (plus the sd_id before the first pair of an element
        // and the "]" / "][" after the last).  Rows are staged behind the cursor in the line's own bytes: slot k ends at
        // sbase + 8 (k + 1) and may be written once the cursor has passed that byte.
        const int sbase = (ls + 7) & ~7;
        unsigned long long* stg = (unsigned long long*)(T + sbase);
        uint32_t n = 0, pairs = 0, hdr = 0;
        int i = d + 1, elem_start = 0, id_end = 0;
        bool st_id = true, active = walk, any_esc = false;
        while (fg_any(active)) {
            if (active && st_id) {  // sd_id: up to the first ' ' (:175-177); any other flagged byte inside it -> slow path
                const uint32_t W = r5_window(bmI, i);
                const int s1 = i + fg_ffs(W) - 1;
                if (W == 0u || s1 >= le || T[s1] != ' ') { ok = false; active = false; }
                else { elem_start = i; id_end = s1; i = s1 + 1; st_id = false; hdr = n++; pairs = 0; }
            }
            // name: unflagged bytes (all legal name characters, :188-192) up to '=' (:208), then '"' (:212)
            int e = i;
            if (active) {
                const uint32_t W = r5_window(bmI, i);
                e = i + fg_ffs(W) - 1;
                if (W == 0u || (W & 1u) || e + 2 >= le || T[e] != '=' || T[e + 1] != '"') { ok = false; active = false; }
            }
            // value: up to the first unescaped '"' (:216, :217, :231).  Every '"' and '\\' is a flagged byte; the flagged
            // bytes of a 32-byte window are walked inside the lane (spaces and the like are stepped over), the warp only
            // loops for values longer than a window.
            int c = e + 2;
            bool has_bs = false;
            {
                bool s = active;
                for (;;) {
                    if (s) {
                        uint32_t W = r5_window(bmI, c);
                        const int room = le - c;  // > 0
                        if (room < 32) W &= (1u << room) - 1u;
                        int adv = 32;
                        while (W) {
                            const int b = fg_ffs(W) - 1;
                            const uint32_t ch = T[c + b];
                            if (ch == '"') { adv = b; s = false; break; }
                            W &= W - 1u;
                            if (ch == '\\') {  // the escaped byte is skipped, whatever it is
                                has_bs = true;
                                W &= ~(2u << b);
                                if (b == 31) adv = 33;
                            }
                        }
                        c += adv;
                        if (s && c >= le) { c = le; s = false; }
                    }
                    if (!fg_any(s)) break;
                }
            }
            if (active) {
                if (c + 1 >= le || sbase + 8 * ((int)n + 1) > c + 1) { ok = false; active = false; }  // :239 / :148 / no room: slow path
                else {
                    stg[n++] = r5_pack_pair8(i - ls, e - ls, c - ls, has_bs);
                    any_esc |= has_bs;
                    ++pairs;
                    const uint32_t nx = T[c + 1];
                    if (nx == ' ') {
                        i = c + 2;
                        if (i >= le) { ok = false; active = false; }
                    } else if (nx == ']') {  // :197 end of this element, then :145-155
                        stg[hdr] = r5_pack_header8(elem_start - ls, id_end - ls, pairs);
                        const uint32_t n2 = c + 2 < le ? T[c + 2] : 0u;
                        if (n2 == ' ') { msg_from = c + 2; active = false; }
                        else if (n2 == '[') { i = c + 3; st_id = true; }
                        else { ok = false; active = false; }
                    } else { ok = false; active = false; }
                }
            }
        }
        if (walk && ok) {
            r.n_entries = n;
            r.stage = stg;
            r.esc = any_esc;
        }
    }

    // ---- parse_msg :163-172, Record assembly :32-47 ------------------------------------------------
    // msg = line[msg_from..].trim(); full_msg = line.trim_end() (:46).  The byte before msg_from is '-' or ']', so when the
    // rest is all whitespace full_msg ends at msg_from.  Common case: the line ends in a plain character and the message
    // starts one space after SD — then no trim loop runs (the votes are warp-wide: every lane gets here).
    int hi = le, lo = msg_from;
    {
        bool plain_end = true, plain_start = true;
        if (ok) {
            const uint32_t cl = T[le - 1];
            plain_end = cl > 0x20u && cl < 0x80u;
            plain_start = false;
            if (msg_from + 1 < le) {
                const uint32_t c0 = T[msg_from], c1 = T[msg_from + 1];
                plain_start = c0 == ' ' && c1 > 0x20u && c1 < 0x80u;
            }
        }
        if (fg_any(!plain_end)) {
            if (ok && !plain_end) hi = trim_end(T, msg_from, le);
        }
        if (fg_any(!plain_start)) {
            if (ok) lo = plain_start ? msg_from + 1 : trim_start(T, msg_from, hi);
        } else {
            lo = msg_from + 1;
        }
    }
    if (ok) {
        if (hi > lo) {
            r.msg_o = lo - ls;
            r.msg_l = hi - lo;
        } else {
            r.msg_o = msg_from - ls;
            r.msg_l = 0;
        }
        r.sp1 = sp[1] - ls;
        r.sp2 = sp[2] - ls;
        r.sp3 = sp[3] - ls;
        r.sp4 = sp[4] - ls;
        r.sp5 = sp[5] - ls;
    }
    fg_syncwarp();
    return ok;
}

}  // namespace fg
