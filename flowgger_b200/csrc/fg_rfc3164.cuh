// fg_rfc3164.cuh — RFC3164Decoder::decode for ONE line (decoder/rfc3164_decoder.rs:31-213), device logic.
//
// The reference tokenises into owned Vecs and re-joins; here a line is walked in place:
//   parse_strip_pri (:126-153)      the '<'..'>' scan at the top of r3164_parse_line
//   decode_rfc_standard (:55-87)    the first six whitespace tokens are located (split_whitespace = Unicode White_Space),
//                                   the date is read off them, then the rest of the line is checked ONCE, four bytes per
//                                   step: if it holds nothing but single ASCII spaces between its tokens the re-joined
//                                   message (`tokens.join(" ")`, :67) IS a span of the input; otherwise the tokens are
//                                   copied, joined by one space, into the arena
//   decode_rfc_custom (:89-123)     two ": " separators; split + join with the same separator is the identity, so the
//                                   message is always a span
//   parse_date (:163-213)           time 0.3 format description "[year] [month repr:short] [day padding:none]
//                                   [hour]:[minute]:[second]" applied to the tokens directly (a token holds no space, the
//                                   description puts one space between its items, so token k must match item k exactly)
//   get_by_name / assume_timezone   tz_find / tz_offset_local over the packed zone table (fg_tz.cu)
// The error returned is that of the last form tried (:40-47).  tests/emu compiles this file with g++.
#pragma once
#include <stdint.h>

#include "fg_common.cuh"
#include "fg_kernels.cuh"
#include "fg_status.h"

#ifdef FG_HOST_EMU
#define FG_HD static inline
#elif defined(__CUDACC__)
#define FG_HD __host__ __device__ __forceinline__
#else
#define FG_HD static inline
#endif

namespace fg {

// ---- zone table ---------------------------------------------------------------------------------------------------
FG_HD unsigned long long tz_fnv1a(const uint8_t* p, int a, int b) {
    unsigned long long h = 0xcbf29ce484222325ull;
    for (int i = a; i < b; ++i) {
        h ^= (unsigned long long)p[i];
        h *= 0x100000001b3ull;
    }
    return h;
}
// get_by_name (exact, case-sensitive): zone of the identifier p[a, b), or -1
FG_HD int tz_find(const TzDeviceTable& T, const uint8_t* p, int a, int b) {
    const int len = b - a;
    if (T.n_names == 0 || len < T.min_len || len > T.max_len) return -1;
    const uint32_t c0 = p[a];
    if (!((T.first_mask[c0 >> 5] >> (c0 & 31u)) & 1u)) return -1;  // ordinary hostnames stop here
    const unsigned long long h = tz_fnv1a(p, a, b);
    int lo = 0, hi = T.n_names;  // first k with hash[k] >= h
    while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if (T.hash[mid] < h) lo = mid + 1;
        else hi = mid;
    }
    for (int k = lo; k < T.n_names && T.hash[k] == h; ++k) {
        const int na = T.name_off[k], nb = T.name_off[k + 1];
        if (nb - na != len) continue;
        bool same = true;
        for (int i = 0; i < len; ++i) same = same && T.names[na + i] == p[a + i];
        if (same) return T.zone[k];
    }
    return -1;
}
// assume_timezone: the UTC offset in force at LOCAL second `local` — the last span whose key is <= local.  fg_tz.cu sets
// key = transition + max(offset before, offset after): a local time that occurs twice takes the earlier offset, one the
// jump skips the offset before the jump.
FG_HD int tz_offset_local(const TzDeviceTable& T, int z, long long local) {
    int lo = T.first[z], hi = T.first[z + 1];
    while (hi - lo > 1) {
        const int mid = (lo + hi) >> 1;
        if (T.key[mid] <= local) lo = mid;
        else hi = mid;
    }
    return T.off[lo];
}

// the line walkers: only the kernel file (and the emulation build) instantiates them; fg_abi.cu / fg_tz.cu use the zone search above
#if defined(FG_HOST_EMU) || (defined(__CUDACC__) && defined(FG_R3164_WALKERS))

struct R3Out {
    uint32_t status, facility, severity, flags;
    double ts;
    int host_o, host_l, msg_o, msg_l, full_l;  // relative to the line start; msg_o indexes the arena with FG_FLAG_MSG_ARENA
};
constexpr uint32_t kR3FlagMsgArena = 0x40u;  // include/flowgger_cuda.h: FG_FLAG_MSG_ARENA

FG_DEV uint32_t r3_ld32(const uint8_t* q) {  // q is 4-byte aligned
#ifdef FG_HOST_EMU
    uint32_t w;
    memcpy(&w, q, 4);
    return w;
#else
    return *reinterpret_cast<const uint32_t*>(q);
#endif
}

// next token of str::split_whitespace at or after pos, inside [pos, end)
FG_DEV bool r3_token(bytes_t p, int& pos, int end, int& a, int& b) {
    while (pos < end) {
        const int w = ws_len_front(p, pos, end);
        if (!w) break;
        pos += w;
    }
    if (pos >= end) return false;
    a = pos;
    while (pos < end) {
        const uint32_t c = p[pos];
        if (c < 0x80u) {
            if (is_ascii_ws(c)) break;
        } else if (ws_len_front(p, pos, end)) {  // a continuation byte never starts a White_Space character
            break;
        }
        ++pos;
    }
    b = pos;
    return true;
}

// [month repr:short], case-sensitive
FG_DEV int r3_month(bytes_t p, int a, int b) {
    if (b - a != 3) return 0;
    const uint32_t k = ((uint32_t)p[a] << 16) | ((uint32_t)p[a + 1] << 8) | (uint32_t)p[a + 2];
    switch (k) {
        case 0x4A616Eu: return 1;   // Jan
        case 0x466562u: return 2;   // Feb
        case 0x4D6172u: return 3;   // Mar
        case 0x417072u: return 4;   // Apr
        case 0x4D6179u: return 5;   // May
        case 0x4A756Eu: return 6;   // Jun
        case 0x4A756Cu: return 7;   // Jul
        case 0x417567u: return 8;   // Aug
        case 0x536570u: return 9;   // Sep
        case 0x4F6374u: return 10;  // Oct
        case 0x4E6F76u: return 11;  // Nov
        case 0x446563u: return 12;  // Dec
        default: return 0;
    }
}
// [year]: optional sign, exactly four digits (time 0.3 without large-dates)
FG_DEV bool r3_year(bytes_t p, int a, int b, int& year) {
    bool neg = false;
    if (a < b && (p[a] == '+' || p[a] == '-')) {
        neg = p[a] == '-';
        ++a;
    }
    if (b - a != 4) return false;
    int i = a, y;
    if (!four_digits(p, i, b, y)) return false;
    year = neg ? -y : y;
    return true;
}
// "[month repr:short] [day padding:none] [hour]:[minute]:[second]" on three tokens + Date::from_calendar_date /
// Time::from_hms -> seconds since the epoch of that civil time read as UTC
FG_DEV bool r3_date(bytes_t p, int year, const int* ta, const int* tb, long long& local) {
    const int month = r3_month(p, ta[0], tb[0]);
    if (!month) return false;
    const int dl = tb[1] - ta[1];
    if (dl < 1 || dl > 2) return false;  // one or two digits, then the separating space
    int day = 0;
    for (int i = ta[1]; i < tb[1]; ++i) {
        const uint32_t d = (uint32_t)p[i] - '0';
        if (d > 9u) return false;
        day = day * 10 + (int)d;
    }
    if (day == 0) return false;  // NonZeroU8
    if (tb[2] - ta[2] != 8) return false;
    int i = ta[2], hh, mm, ss;
    if (!two_digits(p, i, tb[2], hh) || p[i] != ':') return false;
    ++i;
    if (!two_digits(p, i, tb[2], mm) || p[i] != ':') return false;
    ++i;
    if (!two_digits(p, i, tb[2], ss)) return false;
    if (day > days_in_month(year, month)) return false;
    if (hh > 23 || mm > 59 || ss > 59) return false;
    local = (long long)days_from_civil(year, month, day) * 86400 + hh * 3600 + mm * 60 + ss;
    return true;
}

// parse_date_token (:155-161) + parse_date (:163-213) over the first `ntok` (<= 6 known) tokens; idx = tokens consumed
FG_DEV uint32_t r3_parse_date_token(bytes_t p, const R3164DeviceConfig& cfg, int ntok, const int* ta, const int* tb, double& ts,
                                    int& idx) {
    if (ntok < 3) return FG_E3_TIME_FORMAT;
    long long local = 0;
    // without a year: format!("{} {}", current_year, ...) parses only when the year prints as four digits
    bool ok = cfg.year >= 1000 && cfg.year <= 9999 && r3_date(p, cfg.year, ta, tb, local);
    idx = 3;
    if (!ok) {
        if (ntok < 4) return FG_E3_WITH_YEAR;
        int year;
        if (!r3_year(p, ta[0], tb[0], year) || !r3_date(p, year, ta + 1, tb + 1, local)) return FG_E3_DATE;
        idx = 4;
    }
    if (ntok > idx) {
        // (constant indices keep the token arrays in registers)
        const int za = idx == 3 ? ta[3] : ta[4], zb = idx == 3 ? tb[3] : tb[4];
        const int z = tz_find(cfg.tz, p, za, zb);
        if (z >= 0) {
            local -= (long long)tz_offset_local(cfg.tz, z, local);
            idx += 1;
        }
    }
    ts = unix_nanos_to_ts(local, 0u);
    return FG_ST_OK;
}

// true: p[a, b) holds only ASCII bytes >= 0x20 and no two adjacent spaces (so split_whitespace + join(" ") returns it as is,
// given that it neither starts nor ends with a space)
FG_DEV bool r3_plain_run(bytes_t p, int a, int b) {
    bool prev_sp = false;
    int i = a;
    while (i < b && ((size_t)(p + i) & 3u) != 0u) {
        const uint32_t c = p[i];
        if (c < 0x20u || c >= 0x80u) return false;
        const bool sp = c == 0x20u;
        if (sp && prev_sp) return false;
        prev_sp = sp;
        ++i;
    }
    for (; i + 4 <= b; i += 4) {
        const uint32_t w = r3_ld32(p + i);
        if ((w & 0x80808080u) != 0u || ((w - 0x20202020u) & ~w & 0x80808080u) != 0u) return false;  // a byte >= 0x80 or < 0x20
        const uint32_t t = w ^ 0x20202020u;
        const uint32_t z = ~(((t & 0x7F7F7F7Fu) + 0x7F7F7F7Fu) | t) & 0x80808080u;  // bit 8k+7: byte k is a space (exact)
        if ((z & (z >> 8)) != 0u || (prev_sp && (z & 0x80u) != 0u)) return false;
        prev_sp = (z >> 31) != 0u;
    }
    for (; i < b; ++i) {
        const uint32_t c = p[i];
        if (c < 0x20u || c >= 0x80u) return false;
        const bool sp = c == 0x20u;
        if (sp && prev_sp) return false;
        prev_sp = sp;
    }
    return true;
}

// `_log_tokens[1..].join(" ")` (:67) for the text after the hostname token, which ends at `from`; `end` = the line without
// its trailing whitespace
FG_DEV void r3_message(bytes_t p, int from, int end, const R3164DeviceConfig& cfg, R3Out& r) {
    int pos = from, a, b;
    if (!r3_token(p, pos, end, a, b)) {  // no token left: Some("")
        r.msg_o = from;
        r.msg_l = 0;
        return;
    }
    if (r3_plain_run(p, a, end)) {
        r.msg_o = a;
        r.msg_l = end - a;
        return;
    }
    // exact pass: is every gap one ASCII space after all (non-ASCII text, control bytes that are not White_Space)?
    const int first = a;
    bool regular = true;
    uint32_t joined = (uint32_t)(b - a);
    int last_b = b;
    for (;;) {
        int a2, b2;
        if (!r3_token(p, pos, end, a2, b2)) break;
        regular = regular && a2 - last_b == 1 && p[last_b] == 0x20u;
        joined += 1u + (uint32_t)(b2 - a2);
        last_b = b2;
    }
    if (regular) {
        r.msg_o = first;
        r.msg_l = last_b - first;
        return;
    }
    const uint32_t at = atomicAdd(cfg.arena_counter, joined);
    r.msg_o = (int)at;
    r.msg_l = (int)joined;
    r.flags |= kR3FlagMsgArena;
    if ((unsigned long long)at + joined > (unsigned long long)cfg.arena_cap) return;  // the host regrows the arena and redoes the batch
    uint8_t* o = cfg.arena + at;
    pos = first;
    bool lead = true;
    for (;;) {
        int a2, b2;
        if (!r3_token(p, pos, end, a2, b2)) break;
        if (!lead) *o++ = 0x20u;
        lead = false;
        for (int i = a2; i < b2; ++i) *o++ = p[i];
    }
}

// Decoder::decode (:31-48) for the line p[0, len)
FG_DEV void r3164_parse_line(bytes_t p, int len, const R3164DeviceConfig& cfg, R3Out& r) {
    r.status = FG_ST_OK;
    r.facility = r.severity = 0xFFu;
    r.flags = 0u;
    r.ts = 0.0;
    r.host_o = r.msg_o = -1;
    r.host_l = r.msg_l = 0;
    r.full_l = 0;
    // parse_strip_pri (:126-153)
    int m0 = 0;
    if (len > 0 && p[0] == '<') {
        int gt = 1;
        while (gt < len && p[gt] != '>') ++gt;
        if (gt >= len) { r.status = FG_E3_PRI_MALFORMED; return; }
        int a = 0, b = gt + 1;
        while (a < b && p[a] == '<') ++a;       // trim_start_matches('<')
        while (b > a && p[b - 1] == '>') --b;   // trim_end_matches('>')
        uint32_t pri;
        if (!parse_u8(p, a, b, pri)) { r.status = FG_E3_PRI_INVALID; return; }
        r.facility = pri >> 3;
        r.severity = pri & 7u;
        m0 = gt + 1;
    }
    const int end = trim_end(p, 0, len);  // full_msg = line.trim_end() (:77, :112)
    // decode_rfc_standard (:55-87): needs four tokens; the date, an optional zone and the hostname are among the first six
    {
        int ta[6] = {0, 0, 0, 0, 0, 0}, tb[6] = {0, 0, 0, 0, 0, 0}, n = 0, pos = m0;
#pragma unroll
        for (int k = 0; k < 6; ++k)
            if (n == k && r3_token(p, pos, len, ta[k], tb[k])) n = k + 1;
        if (n > 3) {
            double ts;
            int idx;
            if (r3_parse_date_token(p, cfg, n, ta, tb, ts, idx) == FG_ST_OK) {
                if (idx >= n) { r.status = FG_E3_PANIC; return; }  // `_log_tokens[0]` on an empty Vec (:64)
                const int ha = idx == 3 ? ta[3] : (idx == 4 ? ta[4] : ta[5]), hb = idx == 3 ? tb[3] : (idx == 4 ? tb[4] : tb[5]);
                r.ts = ts;
                r.host_o = ha;
                r.host_l = hb - ha;
                r.full_l = end;
                r3_message(p, hb, end, cfg, r);
                return;
            }
        }
    }
    // decode_rfc_custom (:89-123): <hostname>: <date>: <message>
    int s1 = -1, s2 = -1;
    for (int i = m0; i + 1 < len; ++i) {
        if (p[i] == ':' && p[i + 1] == ' ') {
            if (s1 < 0) {
                s1 = i;
                ++i;  // str::split matches do not overlap
            } else {
                s2 = i;
                break;
            }
        }
    }
    if (s2 < 0) { r.status = FG_E3_CUSTOM; return; }
    int ta[5] = {0, 0, 0, 0, 0}, tb[5] = {0, 0, 0, 0, 0}, n = 0, pos = s1 + 2;
#pragma unroll
    for (int k = 0; k < 5; ++k)
        if (n == k && r3_token(p, pos, s2, ta[k], tb[k])) n = k + 1;
    double ts;
    int idx;
    const uint32_t st = r3_parse_date_token(p, cfg, n, ta, tb, ts, idx);
    if (st != FG_ST_OK) { r.status = st; return; }
    r.ts = ts;
    r.host_o = m0;
    r.host_l = s1 - m0;
    r.msg_o = s2 + 2;  // tokens[2..].join(": "): everything behind the second separator, untrimmed
    r.msg_l = len - (s2 + 2);
    r.full_l = end;
}


// ====================================================================================================================
// The same decoder written for a WARP: r3164_parse_lockstep.
//
// With r3164_parse_line above, the 32 lanes of a warp leave each data-dependent loop (PRI digits, token lengths, ...) at
// different iterations and, the function being a thicket of early returns, are not brought back together before its end:
// a few lanes per issued instruction, and the instruction fetch cannot keep up with 32 lanes in 32 places.  Here every lane of the
// warp walks through the SAME sequence of phases; a lane that has nothing to do in a phase idles in it.  Every loop runs
// until no lane of the warp needs another iteration (fg_any), and no lane returns early, so the warp is converged at
// every phase boundary by construction.  The per-lane results are those of r3164_parse_line, statement for statement:
// tests/emu runs both against the oracle (a warp being one lane there, fg_any(p) == p).
//
// All 32 lanes must call this together; `active` = the lane has a line to decode.
// ====================================================================================================================

// The two routines the phases call most are real calls (all lanes make them together): thirteen inlined copies of the
// tokenizer would not fit the instruction cache the warps of an SM share.
#ifdef FG_HOST_EMU
#define FG_LS_CALL static inline
#else
#define FG_LS_CALL static __device__ __noinline__
#endif

// r3_token for the lanes with `want`; the others idle.  Returns whether the lane found a token.
FG_LS_CALL unsigned long long r3_token_pack_ls(bytes_t p, int pos, int end, bool want) {
    bool skip = want;
    while (fg_any(skip)) {
        if (skip) {
            const int w = pos < end ? ws_len_front(p, pos, end) : 0;
            if (w) pos += w;
            else skip = false;
        }
    }
    const bool got = want && pos < end;
    bool run = got;
    const int a = pos;
    while (fg_any(run)) {
        if (run) {
            bool stop = pos >= end;
            if (!stop) {
                const uint32_t c = p[pos];
                stop = c < 0x80u ? is_ascii_ws(c) : ws_len_front(p, pos, end) != 0;
            }
            if (stop) run = false;
            else ++pos;
        }
    }
    // (everything travels by value: references would put the caller's token positions on the stack)
    return got ? ((unsigned long long)(uint32_t)a | ((unsigned long long)(uint32_t)pos << 32)) : 0xFFFFFFFFFFFFFFFFull;
}
// the same with the reference's shape: advances pos past the token (or to `end` when only whitespace was left)
FG_DEV bool r3_token_ls(bytes_t p, int& pos, int end, bool want, int& a, int& b) {
    const unsigned long long t = r3_token_pack_ls(p, pos, end, want);
    const bool got = t != 0xFFFFFFFFFFFFFFFFull;
    if (got) {
        a = (int)(uint32_t)t;
        b = (int)(uint32_t)(t >> 32);
        pos = b;
    } else if (want && pos < end) {
        pos = end;
    }
    return got;
}

// tz_find for the lanes with `want` (-1 for the others and for tokens that are no identifier)
FG_DEV int tz_find_ls(const TzDeviceTable& T, bytes_t p, int a, int b, bool want) {
    const int len = b - a;
    bool cand = want && T.n_names != 0 && len >= T.min_len && len <= T.max_len;
    if (cand) {
        const uint32_t c0 = p[a];
        cand = ((T.first_mask[c0 >> 5] >> (c0 & 31u)) & 1u) != 0u;  // ordinary hostnames stop here
    }
    unsigned long long h = 0xcbf29ce484222325ull;
    int i = a;
    while (fg_any(cand && i < b)) {
        if (cand && i < b) {
            h ^= (unsigned long long)p[i];
            h *= 0x100000001b3ull;
            ++i;
        }
    }
    int lo = 0, hi = T.n_names;  // first k with hash[k] >= h
    while (fg_any(cand && lo < hi)) {
        if (cand && lo < hi) {
            const int mid = (lo + hi) >> 1;
            if (T.hash[mid] < h) lo = mid + 1;
            else hi = mid;
        }
    }
    int z = -1;
    bool look = cand && lo < T.n_names;
    while (fg_any(look)) {  // identifiers with this hash (one, unless two collide)
        if (look) {
            if (lo >= T.n_names || T.hash[lo] != h) {
                look = false;
            } else {
                const int na = T.name_off[lo], nb = T.name_off[lo + 1];
                bool same = nb - na == len;
                for (int q = 0; same && q < len; ++q) same = T.names[na + q] == p[a + q];
                if (same) {
                    z = T.zone[lo];
                    look = false;
                } else {
                    ++lo;
                }
            }
        }
    }
    return z;
}
// tz_offset_local for the lanes with z >= 0
FG_DEV int tz_offset_ls(const TzDeviceTable& T, int z, long long local) {
    int lo = 0, hi = 0;
    if (z >= 0) {
        lo = T.first[z];
        hi = T.first[z + 1];
    }
    while (fg_any(hi - lo > 1)) {
        if (hi - lo > 1) {
            const int mid = (lo + hi) >> 1;
            if (T.key[mid] <= local) lo = mid;
            else hi = mid;
        }
    }
    return z >= 0 ? T.off[lo] : 0;
}

// get_by_name + assume_timezone for the lanes with `want`: the UTC offset at `local`, or kR3NoZone
constexpr long long kR3NoZone = (long long)0x8000000000000000ull;
FG_LS_CALL long long tz_resolve_ls(const TzDeviceTable& T, bytes_t p, int a, int b, bool want, long long local) {
    const int z = tz_find_ls(T, p, a, b, want);
    const int off = tz_offset_ls(T, z, local);
    return z >= 0 ? (long long)off : kR3NoZone;
}
// r3_date by value (no votes inside: may be called by any subset of the lanes); kR3NoZone = the tokens are no date
FG_LS_CALL long long r3_date_v(bytes_t p, int year, int a0, int b0, int a1, int b1, int a2, int b2) {
    const int ta[3] = {a0, a1, a2}, tb[3] = {b0, b1, b2};
    long long local;
    return r3_date(p, year, ta, tb, local) ? local : kR3NoZone;
}

// parse_date_token + parse_date (:155-213) for the lanes with `want`: status (FG_ST_OK: ts and idx are set)
FG_DEV uint32_t r3_parse_date_token_ls(bytes_t p, const R3164DeviceConfig& cfg, bool want, int ntok, const int* ta, const int* tb,
                                       double& ts, int& idx) {
    uint32_t st = FG_ST_OK;
    long long local = 0;
    idx = 3;
    bool ok = false;
    if (want) {
        if (ntok < 3) {
            st = FG_E3_TIME_FORMAT;
        } else {
            if (cfg.year >= 1000 && cfg.year <= 9999) local = r3_date_v(p, cfg.year, ta[0], tb[0], ta[1], tb[1], ta[2], tb[2]);
            else local = kR3NoZone;
            ok = local != kR3NoZone;
            if (!ok) {
                int year;
                if (ntok < 4) st = FG_E3_WITH_YEAR;
                else if (!r3_year(p, ta[0], tb[0], year)) st = FG_E3_DATE;
                else {
                    local = r3_date_v(p, year, ta[1], tb[1], ta[2], tb[2], ta[3], tb[3]);
                    if (local == kR3NoZone) st = FG_E3_DATE;
                    else {
                        ok = true;
                        idx = 4;
                    }
                }
            }
        }
    }
    fg_syncwarp();
    const bool ztry = ok && ntok > idx;
    const int za = idx == 3 ? ta[3] : ta[4], zb = idx == 3 ? tb[3] : tb[4];
    const long long off = tz_resolve_ls(cfg.tz, p, za, zb, ztry, local);
    if (off != kR3NoZone) {
        local -= off;
        idx += 1;
    }
    if (ok) ts = unix_nanos_to_ts(local, 0u);
    fg_syncwarp();
    return want ? st : FG_ST_OK;
}

// r3_plain_run for the lanes with `want`
FG_DEV bool r3_plain_run_ls(bytes_t p, int a, int b, bool want) {
    bool ok = want, prev_sp = false;
    int i = a;
    // bytes up to the next 4-byte boundary (at most three rounds), then words, then the last bytes
    for (int round = 0; round < 3; ++round) {
        if (ok && i < b && ((size_t)(p + i) & 3u) != 0u) {
            const uint32_t c = p[i];
            const bool sp = c == 0x20u;
            if (c < 0x20u || c >= 0x80u || (sp && prev_sp)) ok = false;
            prev_sp = sp;
            ++i;
        }
    }
    while (fg_any(ok && i + 4 <= b)) {
        if (ok && i + 4 <= b) {
            const uint32_t w = r3_ld32(p + i);
            const uint32_t t = w ^ 0x20202020u;
            const uint32_t z = ~(((t & 0x7F7F7F7Fu) + 0x7F7F7F7Fu) | t) & 0x80808080u;  // bit 8k+7: byte k is a space (exact for ASCII)
            if ((w & 0x80808080u) != 0u || ((w - 0x20202020u) & ~w & 0x80808080u) != 0u ||  // a byte >= 0x80 or < 0x20
                (z & (z >> 8)) != 0u || (prev_sp && (z & 0x80u) != 0u))
                ok = false;
            prev_sp = (z >> 31) != 0u;
            i += 4;
        }
    }
    for (int round = 0; round < 3; ++round) {
        if (ok && i < b) {
            const uint32_t c = p[i];
            const bool sp = c == 0x20u;
            if (c < 0x20u || c >= 0x80u || (sp && prev_sp)) ok = false;
            prev_sp = sp;
            ++i;
        }
    }
    return ok;
}

FG_DEV void r3164_parse_lockstep(bytes_t p, int len, bool active, const R3164DeviceConfig& cfg, R3Out& r) {
    r.status = FG_ST_OK;
    r.facility = r.severity = 0xFFu;
    r.flags = 0u;
    r.ts = 0.0;
    r.host_o = r.msg_o = -1;
    r.host_l = r.msg_l = 0;
    r.full_l = 0;
    uint32_t st = FG_ST_OK;
    bool done = !active;  // the lane's result is settled (a Record or an error): it idles through the remaining phases

    // ---- parse_strip_pri (:126-153) ---------------------------------------------------------------------------------
    int m0 = 0;
    {
        const bool has = !done && len > 0 && p[0] == '<';
        bool scan = has;
        int gt = 1;
        while (fg_any(scan)) {
            if (scan) {
                if (gt >= len || p[gt] == '>') scan = false;
                else ++gt;
            }
        }
        if (has) {
            if (gt >= len) {
                st = FG_E3_PRI_MALFORMED;
            } else {
                int a = 0, b = gt + 1;
                while (a < b && p[a] == '<') ++a;      // trim_start_matches('<') (one iteration, unless the line opens with "<<")
                while (b > a && p[b - 1] == '>') --b;  // trim_end_matches('>')
                uint32_t pri;
                if (!parse_u8(p, a, b, pri)) {
                    st = FG_E3_PRI_INVALID;
                } else {
                    r.facility = pri >> 3;
                    r.severity = pri & 7u;
                    m0 = gt + 1;
                }
            }
            done = st != FG_ST_OK;
        }
        fg_syncwarp();
    }
    // ---- line.trim_end() (:77, :112) ----------------------------------------------------------------------------------
    int end = len;
    {
        bool t = !done;
        while (fg_any(t)) {
            if (t) {
                const int w = end > 0 ? ws_len_back(p, 0, end) : 0;
                if (w) end -= w;
                else t = false;
            }
        }
    }
    // ---- decode_rfc_standard (:55-87) ---------------------------------------------------------------------------------
    {
        int ta[6] = {0, 0, 0, 0, 0, 0}, tb[6] = {0, 0, 0, 0, 0, 0}, n = 0, pos = m0;
#pragma unroll
        for (int k = 0; k < 6; ++k)
            if (r3_token_ls(p, pos, len, !done && n == k, ta[k], tb[k])) n = k + 1;
        const bool stry = !done && n > 3;
        double ts = 0.0;
        int idx = 3;
        const uint32_t dst = r3_parse_date_token_ls(p, cfg, stry, n, ta, tb, ts, idx);
        const bool dated = stry && dst == FG_ST_OK;
        if (dated && idx >= n) {  // `_log_tokens[0]` on an empty Vec (:64)
            st = FG_E3_PANIC;
            done = true;
        }
        const bool rec = dated && !done;
        const int ha = idx == 3 ? ta[3] : (idx == 4 ? ta[4] : ta[5]), hb = idx == 3 ? tb[3] : (idx == 4 ? tb[4] : tb[5]);
        if (rec) {
            r.ts = ts;
            r.host_o = ha;
            r.host_l = hb - ha;
            r.full_l = end;
        }
        // `_log_tokens[1..].join(" ")` (:67)
        int mpos = hb, ma = 0, mb = 0;
        const bool got = r3_token_ls(p, mpos, end, rec, ma, mb);
        if (rec && !got) {  // no token left: Some("")
            r.msg_o = hb;
            r.msg_l = 0;
        }
        const bool chk = rec && got;
        const bool plain = r3_plain_run_ls(p, ma, end, chk);
        if (chk && plain) {
            r.msg_o = ma;
            r.msg_l = end - ma;
        }
        // exact pass: is every gap one ASCII space after all?
        const bool slow = chk && !plain;
        bool regular = true, more = slow;
        uint32_t joined = (uint32_t)(mb - ma);
        int last_b = mb;
        while (fg_any(more)) {
            int a2 = 0, b2 = 0;
            const bool g2 = r3_token_ls(p, mpos, end, more, a2, b2);
            if (g2) {
                regular = regular && a2 - last_b == 1 && p[last_b] == 0x20u;
                joined += 1u + (uint32_t)(b2 - a2);
                last_b = b2;
            }
            more = g2;
        }
        if (slow && regular) {
            r.msg_o = ma;
            r.msg_l = last_b - ma;
        }
        const bool join = slow && !regular;
        uint32_t at = 0;
        if (join) {
            at = atomicAdd(cfg.arena_counter, joined);
            r.msg_o = (int)at;
            r.msg_l = (int)joined;
            r.flags |= kR3FlagMsgArena;
        }
        fg_syncwarp();
        const bool copy = join && (unsigned long long)at + joined <= (unsigned long long)cfg.arena_cap;  // else: the host regrows and redoes
        uint8_t* o = cfg.arena + at;
        int cpos = ma;
        bool lead = true;
        more = copy;
        while (fg_any(more)) {
            int a2 = 0, b2 = 0;
            const bool g2 = r3_token_ls(p, cpos, end, more, a2, b2);
            if (g2 && !lead) *o++ = 0x20u;
            if (g2) lead = false;
            int q = a2;
            while (fg_any(g2 && q < b2)) {
                if (g2 && q < b2) *o++ = p[q++];
            }
            more = g2;
        }
        if (rec) done = true;
    }
    // ---- decode_rfc_custom (:89-123): <hostname>: <date>: <message> ----------------------------------------------------
    {
        const bool cus = !done;
        int s1 = -1, s2 = -1, i = m0;
        bool sc = cus;
        while (fg_any(sc)) {
            if (sc) {
                if (i + 1 >= len) {
                    sc = false;
                } else if (p[i] == ':' && p[i + 1] == ' ') {
                    if (s1 < 0) {
                        s1 = i;
                        i += 2;  // str::split matches do not overlap
                    } else {
                        s2 = i;
                        sc = false;
                    }
                } else {
                    ++i;
                }
            }
        }
        if (cus && s2 < 0) {
            st = FG_E3_CUSTOM;
            done = true;
        }
        const bool ctry = cus && !done;
        int ta[5] = {0, 0, 0, 0, 0}, tb[5] = {0, 0, 0, 0, 0}, n = 0, pos = s1 + 2;
#pragma unroll
        for (int k = 0; k < 5; ++k)
            if (r3_token_ls(p, pos, s2, ctry && n == k, ta[k], tb[k])) n = k + 1;
        double ts = 0.0;
        int idx = 3;
        const uint32_t dst = r3_parse_date_token_ls(p, cfg, ctry, n, ta, tb, ts, idx);
        if (ctry) {
            if (dst != FG_ST_OK) {
                st = dst;
            } else {
                r.ts = ts;
                r.host_o = m0;
                r.host_l = s1 - m0;
                r.msg_o = s2 + 2;  // tokens[2..].join(": "): everything behind the second separator, untrimmed
                r.msg_l = len - (s2 + 2);
                r.full_l = end;
            }
        }
    }
    r.status = st;
    fg_syncwarp();
}

#endif  // FG_HOST_EMU || FG_R3164_WALKERS

}  // namespace fg
