// fg_ltsvfast.cuh — LTSV on the bitmap pipeline, PART-parallel: the tab-separated parts of a line are independent of each
// other, so the unit of work of the hot phase is a part, not a line.
//
// H100-native replacement for LTSVDecoder::decode (flowgger src/flowgger/decoder/ltsv_decoder.rs:87-221); the
// value parsers (parse_ts :263-267, the typed schema values :138-195) are the ones of fg_ltsv.cuh, called on tile bytes.
//
//   stage 1  lt_tab16: every thread takes 32-byte granules of the flat tile (two LDS.128, all 32 lanes busy) and writes one
//            word of the TAB bitmap T (line.split('\t') :94), exact per byte.
//   tabs     one thread per line lists the positions of its TABs (find-first-set over T) into the line's slots: slot k of a
//            line = its k-th part, ending at tabs[k] (the last one at the end of the line).  #slots = #tabs + 1.
//   parts    lt_part: one thread per SLOT, for all slots of the CTA round, 256 threads wide: the key ends at the first ':'
//            (splitn(2, ':') :95, a SWAR test on the first 8 key bytes), the four reserved keys are recognised from
//            those 8 bytes, everything else becomes a packed side-table row in the slot.  No loop over a line, no lock step,
//            no lane waits for a longer line (a thread-per-line walk makes every lane wait for the warp's longest line).
//   lines    lt_finish_line: one thread per line parses the (last) `time` and `level` values, picks the first failing part
//            and builds the row.
// Lines that need the reference's sequential semantics beyond that — a repeated `time` or `level` key — and lines that do
// not fit the tile or the slots go through the round-1 scanner (fg_ltsv.cuh), one at a time.
#pragma once
#include "fg_common.cuh"
#include "fg_ltsv.cuh"
#include "fg_r5fast.cuh"
#include "fg_status.h"

namespace fg {

// ---- stage 1 ----------------------------------------------------------------------------------------------------
// 0x80 in every byte of w that equals the byte replicated in pat; exact per byte (no cross-byte carries)
FG_DEV uint32_t lt_eq_flags(uint32_t w, uint32_t pat) {
    const uint32_t x = w ^ pat;
    const uint32_t y = ((x & 0x7F7F7F7Fu) + 0x7F7F7F7Fu) | x;  // bit 7: byte != 0
    return ~y & 0x80808080u;
}
FG_DEV uint32_t lt_tab16(uint32_t w0, uint32_t w1, uint32_t w2, uint32_t w3) {
    return r5_gather16(lt_eq_flags(w0, 0x09090909u), lt_eq_flags(w1, 0x09090909u), lt_eq_flags(w2, 0x09090909u), lt_eq_flags(w3, 0x09090909u));
}

// TABs inside tile range [ls, le)
FG_DEV int lt_count_tabs(const uint32_t* bmT, int ls, int le) {
    if (le <= ls) return 0;
    const int w0 = ls >> 5, w1 = (le - 1) >> 5;
    int cnt = 0;
    for (int w = w0; w <= w1; ++w) {
        uint32_t m = bmT[w];
        if (w == w0) m &= 0xFFFFFFFFu << (ls & 31);
        if (w == w1 && (le & 31)) m &= 0xFFFFFFFFu >> (32 - (le & 31));
        cnt += __popc(m);
    }
    return cnt;
}

// staged side-table row: key start (tile-relative) | key length << 16 | value length << 32 | meta << 56; the value starts
// one byte after the key (the colon).  meta = fg_ltsv_type | FG_EM_SUFFIX | kLtRow (the slot holds a row); typed values
// sit in the parallel `stage_val`.  A slot without a row (reserved key, part without ':') is 0.
constexpr uint32_t kLtRow = 0x80u;
FG_DEV unsigned long long lt_pack_entry(int ka, int kn, int vl, uint32_t meta) {
    return (unsigned long long)(uint32_t)ka | ((unsigned long long)(uint32_t)kn << 16) | ((unsigned long long)(uint32_t)vl << 32) |
           ((unsigned long long)meta << 56);
}

// ---- stage 2 ----------------------------------------------------------------------------------------------------
// the first 8 bytes at p (any alignment), little-endian; reads up to 11 bytes past p (tile + bitmaps are contiguous)
FG_DEV unsigned long long lt_load8(const uint8_t* p) {
#ifdef FG_HOST_EMU
    unsigned long long v;
    memcpy(&v, p, 8);
    return v;
#else
    const uint32_t sh = ((uint32_t)(size_t)p & 3u) * 8u;
    const uint32_t* w = reinterpret_cast<const uint32_t*>(p - ((size_t)p & 3u));
    const uint32_t w0 = w[0], w1 = w[1], w2 = w[2];
    return (unsigned long long)__funnelshift_r(w0, w1, sh) | ((unsigned long long)__funnelshift_r(w1, w2, sh) << 32);
#endif
}

// The schema (ltsv_decoder.rs:19-22) as the walker reads it: from shared memory when the kernel staged it (`names` etc.
// then point into the CTA's copy), with two cheap filters in front of the byte compares — a key can only be a schema key
// if its length and its first byte occur in the schema.
struct LtsvSchemaView {
    const uint8_t* names;
    const int32_t* name_off;
    const int32_t* types;
    int n;
    uint32_t len_mask;        // bit min(len, 31)
    const uint32_t* first;    // [8] 256-bit set of first bytes (nullptr: no filter)
};
// the two filters of a schema (one thread)
FG_DEV void lt_schema_filters(const uint8_t* names, const int32_t* name_off, int n, uint32_t& len_mask, uint32_t* first /* [8] */) {
    len_mask = 0;
    for (int k = 0; k < 8; ++k) first[k] = 0;
    for (int k = 0; k < n; ++k) {
        const int o = name_off[k], l = name_off[k + 1] - o;
        len_mask |= 1u << (l < 31 ? l : 31);
        if (l > 0) first[names[o] >> 5] |= 1u << (names[o] & 31u);
    }
}
FG_DEV int lt_schema_type(bytes_t p, int a, int n, unsigned long long k8, const LtsvSchemaView& S) {
    if (!((S.len_mask >> (n < 31 ? n : 31)) & 1u)) return 0;
    if (S.first != nullptr && n > 0) {
        const uint32_t c = (uint32_t)(k8 & 0xFFu);
        if (!((S.first[c >> 5] >> (c & 31u)) & 1u)) return 0;
    }
    for (int k = 0; k < S.n; ++k) {
        const int o = S.name_off[k], l = S.name_off[k + 1] - o;
        if (l != n) continue;
        bool eq = true;
        for (int j = 0; j < n && eq; ++j) eq = S.names[o + j] == p[a + j];
        if (eq) return S.types[k];
    }
    return 0;
}

// positions of the TABs of [ls, le) into tabs[0 .. n - 1), tabs[n - 1] = le; n = #tabs + 1 (the caller reserved n slots)
FG_DEV void lt_list_tabs(const uint32_t* bmT, int ls, int le, uint16_t* tabs) {
    int k = 0;
    if (le > ls) {
        const int w0 = ls >> 5, w1 = (le - 1) >> 5;
        for (int w = w0; w <= w1; ++w) {
            uint32_t m = bmT[w];
            if (w == w0) m &= 0xFFFFFFFFu << (ls & 31);
            if (w == w1 && (le & 31)) m &= 0xFFFFFFFFu >> (32 - (le & 31));
            while (m) {
                tabs[k++] = (uint16_t)((w << 5) + fg_ffs(m) - 1);
                m &= m - 1u;
            }
        }
    }
    tabs[k] = (uint16_t)le;
}

// 0x80 in every byte of the 8 that is ':'
FG_DEV unsigned long long lt_colon_flags8(unsigned long long k8) {
    const uint32_t lo = lt_eq_flags((uint32_t)k8, 0x3A3A3A3Au), hi = lt_eq_flags((uint32_t)(k8 >> 32), 0x3A3A3A3Au);
    return (unsigned long long)lo | ((unsigned long long)hi << 32);
}
FG_DEV int lt_first_flag8(unsigned long long z) {  // byte index of the lowest 0x80 flag (z != 0)
    const uint32_t lo = (uint32_t)z;
    return lo ? (fg_ffs(lo) - 1) >> 3 : 4 + ((fg_ffs((uint32_t)(z >> 32)) - 1) >> 3);
}

enum { LP_NONE = 0 /* no ':' */, LP_ROW, LP_HOST, LP_MSG, LP_TIME, LP_LEVEL };
struct LtPart {
    int kind;
    int kn;                    // key length: key = [start, start + kn), value = [start + kn + 1, end)
    unsigned long long row;    // LP_ROW: the packed side-table row (typed values: parsed later by lt_typed_value)
};

// One tab-separated part [start, end) of the tile (:95-199 without the value parsers).
template <bool TYPED>
FG_DEV LtPart lt_part(const uint8_t* T, int start, int end, const LtsvDeviceConfig& cfg, const LtsvSchemaView& S) {
    LtPart r;
    r.kind = LP_NONE;
    r.kn = 0;
    r.row = 0;
    const int len = end - start;
    const unsigned long long k8 = lt_load8(T + start);
    int kn = -1;
    {
        const unsigned long long z = lt_colon_flags8(k8);
        if (z) {
            const int b = lt_first_flag8(z);
            if (b < len) kn = b;
        } else {
            for (int i = 8; i < len && kn < 0; i += 8) {  // keys of 8 bytes and more
                const unsigned long long z2 = lt_colon_flags8(lt_load8(T + start + i));
                if (z2) {
                    const int b = i + lt_first_flag8(z2);
                    if (b < len) kn = b;
                    break;
                }
            }
        }
    }
    if (kn < 0) return r;  // println! "Missing value" :99
    r.kn = kn;
    const uint32_t k4 = (uint32_t)k8;
    if (kn == 4 && k4 == 0x656D6974u) r.kind = LP_TIME;                                                     // "time"  :104
    else if (kn == 4 && k4 == 0x74736F68u) r.kind = LP_HOST;                                                // "host"
    else if (kn == 7 && (k8 & 0x00FFFFFFFFFFFFFFull) == 0x006567617373656Dull) r.kind = LP_MSG;             // "message"
    else if (kn == 5 && (k8 & 0x000000FFFFFFFFFFull) == 0x0000006C6576656Cull) r.kind = LP_LEVEL;           // "level"  :114
    else {
        r.kind = LP_ROW;
        uint32_t meta = kLtRow;
        if (TYPED) {
            const int type = lt_schema_type(T, start, kn, k8, S);
            if (type != 0) {
                meta |= (uint32_t)type;  // FG_TAG_* == fg_ltsv_type
                if (ltsv_needs_suffix(T, start, kn, type, cfg)) meta |= 0x20u;  // FG_EM_SUFFIX
            }
        }
        r.row = lt_pack_entry(start, kn, len - kn - 1, meta);
    }
    return r;
}

// which of parse_ts's four attempts (:263-267) will most likely take the value [a, b): only a SCHEDULING hint — lanes with
// the same class run ltsv_parse_ts side by side, the result never depends on it.  0 other, 1 decimal, 2 RFC3339, 3 English.
FG_DEV int lt_time_class(const uint8_t* T, int a, int b) {
    if (b - a >= 2 && T[a] == '[' && T[b - 1] == ']') { ++a; --b; }
    if (b - a < 4) return (b > a && is_digit(T[a])) ? 1 : 0;
    if (T[a + 1] == '/' || T[a + 2] == '/') return 3;
    if (b - a > 10 && T[a + 4] == '-' && (T[a + 10] | 0x20u) == 't') return 2;
    return is_digit(T[a]) || T[a] == '.' || T[a] == '-' || T[a] == '+' ? 1 : 0;
}
// `time` value [a, b) -> Record.ts (:104-111)
FG_DEV bool lt_time_value(const uint8_t* T, int a, int b, double& ts) {
    if (b - a >= 2 && T[a] == '[' && T[b - 1] == ']') { ++a; --b; }  // :105-109
    return ltsv_parse_ts(T, a, b, ts);
}

// the reference's per-line rules once every part is classified (:104-121, :205-219).  t_k = index of the only `time` part
// (t_k < 0: none), ts_ok / ts = what lt_time_value made of its value; l_a / l_b / l_k = the value of the only `level` part
// (l_a < 0: none) and its index; err_in = the smallest (part index << 8 | status) among the typed values that failed
// (0xFFFFFFFF: none).  Fills ts / severity / status; returns the index of the failing part (or -1).
FG_DEV int lt_finish_line(const uint8_t* T, int t_k, bool ts_ok, double ts, int l_a, int l_b, int l_k, uint32_t err_in, bool have_host,
                          LineResult& r) {
    uint32_t err = err_in;
    bool have_ts = false;
    if (t_k >= 0 && (uint32_t)t_k < (err >> 8)) {
        if (ts_ok) { r.ts = ts; have_ts = true; }
        else err = ((uint32_t)t_k << 8) | FG_EL_TS;
    }
    if (l_a >= 0 && (uint32_t)l_k < (err >> 8)) {
        uint32_t sev;
        if (!parse_u8(T, l_a, l_b, sev)) err = ((uint32_t)l_k << 8) | FG_EL_SEV;
        else if (sev > 7u) err = ((uint32_t)l_k << 8) | FG_EL_SEV_HIGH;
        else r.severity = sev;
    }
    if (err != 0xFFFFFFFFu) {
        r.status = err & 0xFFu;
        return (int)(err >> 8);
    }
    if (!have_ts) r.status = FG_EL_MISSING_TS;          // :205
    else if (!have_host) r.status = FG_EL_MISSING_HOST;  // :206
    else r.status = FG_ST_OK;
    return -1;
}

// rows among the slots [lo, hi) of a round: mask word w holds the row bits of slots [32 w, 32 w + 32)
FG_DEV uint32_t lt_rows_between(const uint32_t* mask, uint32_t lo, uint32_t hi) {
    if (hi <= lo) return 0u;
    const uint32_t w0 = lo >> 5, w1 = (hi - 1u) >> 5;
    uint32_t n = 0;
    for (uint32_t w = w0; w <= w1; ++w) {
        uint32_t m = mask[w];
        if (w == w0) m &= 0xFFFFFFFFu << (lo & 31u);
        if (w == w1 && (hi & 31u)) m &= 0xFFFFFFFFu >> (32u - (hi & 31u));
        n += (uint32_t)__popc(m);
    }
    return n;
}

}  // namespace fg
