// fg_gelffast.cuh — GELF on the bitmap pipeline, MEMBER-parallel, for REGULAR lines; everything else goes to the exact
// parser of fg_gelf.cuh.
//
// H100-native replacement for GelfDecoder::decode (flowgger src/flowgger/decoder/gelf_decoder.rs:34-125).  A regular
// line is what every GELF sender emits: ONE flat JSON object
//     { "key" : value , "key" : value ... }        value = string | number | true | false | null
// with nothing but spaces between the tokens, no escape inside a key, no raw control byte anywhere, at most
// kMaxLocalMembers members.  The shape is PROVEN here — with serde_json's own rules for what it accepts (string escapes
// incl. \uXXXX surrogate pairs: read.rs parse_escape; numbers: json_number of fg_gelf.cuh) — and the first byte that does
// not fit (a nested container, a TAB or LF between tokens, a raw control byte, any syntax error ...) hands the line to
// gelf_parse_line, which restates the whole grammar, the newline retry of :44-46 and every error string.  A line accepted
// here is parsed to exactly the members the full parser would collect.
//
//   stage 1  gf_bits16: every thread takes 32-byte granules of the flat tile and writes one word each of three bitmaps,
//            exact per byte — Q '"', B '\\', P ',' — plus one bit per granule "holds a byte < 0x20".
//   lines    gf_line_members: one thread per line runs over the line's bitmap WORDS (17 for 520 bytes, not over its bytes):
//            backslash runs -> escaped quotes -> string interior by a prefix XOR (the simdjson recipe on 32-bit words);
//            the commas outside strings end the members and are listed into the line's slots.
//   members  gf_member: one thread per MEMBER, for all members of the CTA round, 256 threads wide: key, colon, value token,
//            string escapes, literals; numbers are listed and go through json_number in a dense second pass.
//   phase 2  gf_finish: one thread per line sorts the members by key (8-byte prefix first), keeps the last duplicate and
//            applies the per-key rules of gelf_decoder.rs:51-107.
// (Walking a line member by member in lock step — the first two versions — was slower than the round-1 tokenizer.)
#pragma once
#include "fg_common.cuh"
#include "fg_gelf.cuh"
#include "fg_ltsvfast.cuh"  // lt_eq_flags, lt_load8
#include "fg_r5fast.cuh"
#include "fg_status.h"

namespace fg {

// ---- stage 1 ----------------------------------------------------------------------------------------------------
// 16 bytes -> 16 bits of Q, B, P each; ctrl = nonzero iff one of the 16 bytes is < 0x20
FG_DEV void gf_bits16(uint32_t w0, uint32_t w1, uint32_t w2, uint32_t w3, uint32_t& q, uint32_t& b, uint32_t& p, uint32_t& ctrl) {
    q = r5_gather16(lt_eq_flags(w0, 0x22222222u), lt_eq_flags(w1, 0x22222222u), lt_eq_flags(w2, 0x22222222u), lt_eq_flags(w3, 0x22222222u));
    b = r5_gather16(lt_eq_flags(w0, 0x5C5C5C5Cu), lt_eq_flags(w1, 0x5C5C5C5Cu), lt_eq_flags(w2, 0x5C5C5C5Cu), lt_eq_flags(w3, 0x5C5C5C5Cu));
    p = r5_gather16(lt_eq_flags(w0, 0x2C2C2C2Cu), lt_eq_flags(w1, 0x2C2C2C2Cu), lt_eq_flags(w2, 0x2C2C2C2Cu), lt_eq_flags(w3, 0x2C2C2C2Cu));
    ctrl = lt_eq_flags(w0 & 0xE0E0E0E0u, 0u) | lt_eq_flags(w1 & 0xE0E0E0E0u, 0u) | lt_eq_flags(w2 & 0xE0E0E0E0u, 0u) | lt_eq_flags(w3 & 0xE0E0E0E0u, 0u);
}

// ---- stage 2 ----------------------------------------------------------------------------------------------------
FG_DEV bool gf_hex4(const uint8_t* T, int at, uint32_t& n) {
    n = 0;
    for (int k = 0; k < 4; ++k) {
        const uint32_t c = T[at + k];
        uint32_t v;
        if (c - '0' <= 9u) v = c - '0';
        else if ((c | 0x20u) - 'a' <= 5u) v = (c | 0x20u) - 'a' + 10u;
        else return false;
        n = n * 16u + v;
    }
    return true;
}
// h = position of a backslash inside a string: position after the whole escape sequence (read.rs parse_escape), or -1 when
// serde_json rejects it (the exact parser then reports the error)
FG_DEV int gf_escape_end(const uint8_t* T, int h, int le) {
    if (h + 1 >= le) return -1;
    const uint32_t x = T[h + 1];
    if (x == '"' || x == '\\' || x == '/' || x == 'b' || x == 'f' || x == 'n' || x == 'r' || x == 't') return h + 2;
    if (x != 'u') return -1;
    uint32_t n1;
    if (h + 6 > le || !gf_hex4(T, h + 2, n1)) return -1;
    if (n1 >= 0xDC00u && n1 <= 0xDFFFu) return -1;  // LoneLeadingSurrogateInHexEscape
    if (n1 >= 0xD800u && n1 <= 0xDBFFu) {
        uint32_t n2;
        if (h + 12 > le || T[h + 6] != '\\' || T[h + 7] != 'u' || !gf_hex4(T, h + 8, n2)) return -1;
        if (n2 < 0xDC00u || n2 > 0xDFFFu) return -1;
        return h + 12;
    }
    return h + 6;
}

// GKEY_* of a raw key (keys with escapes never get here): the six keys gelf_decoder.rs:51-96 consumes, else GKEY_OTHER
FG_DEV int gf_key_kind(const uint8_t* k, int len) {
    const unsigned long long a = lt_load8(k), b = lt_load8(k + 8);
    switch (len) {
        case 4: return (uint32_t)a == 0x74736F68u ? GKEY_HOST : GKEY_OTHER;
        case 5: return (a & 0x000000FFFFFFFFFFull) == 0x0000006C6576656Cull ? GKEY_LEVEL : GKEY_OTHER;
        case 7: return (a & 0x00FFFFFFFFFFFFFFull) == 0x006E6F6973726576ull ? GKEY_VERSION : GKEY_OTHER;
        case 9: return (a == 0x6D617473656D6974ull && (b & 0xFFull) == 0x70ull) ? GKEY_TIMESTAMP : GKEY_OTHER;              // timestam|p
        case 12: return (a == 0x73656D5F6C6C7566ull && (uint32_t)b == 0x65676173u) ? GKEY_FULL : GKEY_OTHER;                // full_mes|sage
        case 13: return (a == 0x656D5F74726F6873ull && (b & 0x000000FFFFFFFFFFull) == 0x0000006567617373ull) ? GKEY_SHORT : GKEY_OTHER;  // short_me|ssage
        default: return GKEY_OTHER;
    }
}
// the first 8 key bytes as a big-endian number, zero-padded: orders like the bytes do (key bytes are never 0)
FG_DEV unsigned long long gf_key_prefix(const uint8_t* k, int len) {
    unsigned long long a = lt_load8(k);
    if (len < 8) a &= (1ull << (8 * len)) - 1ull;
    const uint32_t lo = (uint32_t)a, hi = (uint32_t)(a >> 32);
#ifdef FG_HOST_EMU
    return ((unsigned long long)__builtin_bswap32(lo) << 32) | __builtin_bswap32(hi);
#else
    return ((unsigned long long)__byte_perm(lo, 0u, 0x0123) << 32) | __byte_perm(hi, 0u, 0x0123);
#endif
}

// ---- lines: member boundaries from the bitmap words ----------------------------------------------------------------
// bits of w below position `lo` / at and above `hi` (positions inside the word's 32) cleared
FG_DEV uint32_t gf_clip(uint32_t w, int word, int lo, int hi) {
    const int base = word << 5;
    if (lo > base) w &= 0xFFFFFFFFu << (lo - base);
    if (hi < base + 32) w &= hi > base ? 0xFFFFFFFFu >> (base + 32 - hi) : 0u;
    return w;
}
// The structural commas of the line [ls, le) — commas outside strings — as tile positions into cuts[0 .. n), n <= cap;
// returns n, or -1 when the line is not regular on this level: a string that does not close, more commas than `cap`.
// The recipe per 32-bit word (simdjson's, with the carries kept in two registers): backslashes that start an odd-length run
// escape the byte behind the run; quotes that are not escaped toggle "inside a string"; a prefix XOR spreads that over the
// word.
FG_DEV int gf_line_commas(const uint32_t* bmQ, const uint32_t* bmB, const uint32_t* bmP, int ls, int le, uint16_t* cuts, int cap, bool act) {
    // All lanes of the warp call (act = this lane has a line): the word loop and the comma loop run in lock step — written
    // with plain loops and early returns the lanes of a warp drifted apart and ran one at a time.
    const bool run = act && le > ls;
    const int w0 = ls >> 5, w1 = run ? (le - 1) >> 5 : w0 - 1;
    uint32_t prev_escaped = 0u;    // bit 0: the first byte of this word is escaped by a run ending in the previous word
    uint32_t prev_in_string = 0u;  // all ones: the previous word ended inside a string
    int n = 0;
    bool bad = false;
    for (int w = w0; fg_any(w <= w1); ++w) {
        uint32_t c = 0u;
        if (w <= w1) {
            uint32_t bs = gf_clip(bmB[w], w, ls, le);
            const uint32_t q = gf_clip(bmQ[w], w, ls, le), pc = gf_clip(bmP[w], w, ls, le);
            // escaped bytes
            bs &= ~prev_escaped;
            const uint32_t follows = (bs << 1) | prev_escaped;
            const uint32_t odd_starts = bs & ~0x55555555u & ~follows;
            const uint32_t sum = odd_starts + bs;
            prev_escaped = sum < odd_starts ? 1u : 0u;  // a run reaching the end of the word that started on an odd bit
            const uint32_t escaped = (0x55555555u ^ (sum << 1)) & follows;
            // string interior
            uint32_t x = q & ~escaped;
            x ^= x << 1;
            x ^= x << 2;
            x ^= x << 4;
            x ^= x << 8;
            x ^= x << 16;
            x ^= prev_in_string;
            prev_in_string = (uint32_t)((int32_t)x >> 31);
            c = pc & ~x;
        }
        for (;;) {
            const bool more = c != 0u;
            if (!fg_any(more)) break;
            if (more) {
                if (n < cap) cuts[n] = (uint16_t)((w << 5) + fg_ffs(c) - 1);
                else bad = true;
                ++n;
                c &= c - 1u;
            }
        }
    }
    return (bad || prev_in_string) ? -1 : n;
}

// the line [ls, le) as member spans: returns the number of members m (their spans are [start_k, cuts[k]) with
// start_0 = `open` + 1, start_k = cuts[k - 1] + 1, the last cut being the closing brace), or -1: not regular.
FG_DEV int gf_line_members(const uint8_t* T, const uint32_t* bmQ, const uint32_t* bmB, const uint32_t* bmP, int ls, int le, uint16_t* cuts,
                           int cap, int& open, bool act) {
    int a = ls, b = le;
    for (;;) {
        const bool m = act && a < b && T[a] == ' ';
        if (!fg_any(m)) break;
        if (m) ++a;
    }
    for (;;) {
        const bool m = act && b > a && T[b - 1] == ' ';
        if (!fg_any(m)) break;
        if (m) --b;
    }
    const bool shape = act && b - a >= 2 && T[a] == '{' && T[b - 1] == '}';
    open = a;
    const int n = gf_line_commas(bmQ, bmB, bmP, a + 1, b - 1, cuts, cap - 1, shape);
    if (!shape || n < 0) return -1;
    if (n == 0) {  // `{}` or one member
        int c = a + 1;
        while (c < b - 1 && T[c] == ' ') ++c;
        if (c == b - 1) return 0;
    }
    cuts[n] = (uint16_t)(b - 1);
    return n + 1;
}

// does [ls, le) hold a byte < 0x20?  anyK has one bit per 32-byte granule ("some byte of the granule is < 0x20"); only the
// flagged granules are looked at byte by byte (in split mode those are the two that hold line terminators)
FG_DEV bool gf_has_ctrl(const uint8_t* T, const uint32_t* anyK, int ls, int le) {
    if (le <= ls) return false;
    const int g0 = ls >> 5, g1 = (le - 1) >> 5;
    for (int g = g0; g <= g1; ++g) {
        if (!((anyK[g >> 5] >> (g & 31)) & 1u)) continue;
        const int a = g == g0 ? ls : g << 5, b = g == g1 ? le : (g << 5) + 32;
        for (int i = a; i < b; ++i)
            if (T[i] < 0x20u) return true;
    }
    return false;
}

// ---- members ---------------------------------------------------------------------------------------------------------
// Everything below is called by ALL lanes of a warp (act = this lane has work) and loops in lock step.
// position of the first set bit of bm in [from, to), or -1
FG_DEV int gf_next_bit(const uint32_t* bm, int from, int to, bool act) {
    const bool run = act && from < to;
    int w = from >> 5;
    uint32_t m = run ? bm[w] & (0xFFFFFFFFu << (from & 31)) : 0u;
    for (;;) {
        const bool more = run && m == 0u && ((w + 1) << 5) < to;
        if (!fg_any(more)) break;
        if (more) m = bm[++w];
    }
    if (m == 0u) return -1;
    const int h = (w << 5) + fg_ffs(m) - 1;
    return h < to ? h : -1;
}
// is the byte at h escaped, i.e. preceded by an odd number of backslashes?  (the byte before the string body is its
// opening quote, so the run cannot reach back past it)
FG_DEV bool gf_escaped(const uint32_t* bmB, int h) {
    const int s0 = h >= 32 ? h - 32 : 0, nb = h - s0;
    if (nb == 0) return false;
    const uint32_t W = r5_window(bmB, s0) << (32 - nb);  // bit 31 = the byte before h
    int run = fg_clz(~W);
    if (run >= nb && nb == 32) {  // 32 backslashes and more: count on
        for (int i = s0 - 1; i >= 0 && ((bmB[i >> 5] >> (i & 31)) & 1u); --i) ++run;
    }
    return (run & 1) != 0;
}
FG_DEV void gf_skip_spaces(const uint8_t* T, int& p, int b, bool act) {
    for (;;) {
        const bool m = act && p < b && T[p] == ' ';
        if (!fg_any(m)) break;
        if (m) ++p;
    }
}

constexpr uint32_t kGfNumber = 0xFFu;  // meta of a member whose number token still has to go through json_number

// One member [a, b) of a regular-looking line: validates it the way serde_json does and produces the member as the exact
// parser would (name span absolute, value, tag | flags | key class << 5).  A number is only located: its token span is
// left in `val` with meta = kGfNumber (gf_member_number finishes it).  false: the line is not regular.
FG_DEV bool gf_member(const uint8_t* T, const uint32_t* bmQ, const uint32_t* bmB, int a, int b, int line_off, int ls, bool act, int2& name,
                      unsigned long long& val, uint32_t& meta) {
    bool ok = act;
    gf_skip_spaces(T, a, b, ok);
    for (;;) {
        const bool m = ok && b > a && T[b - 1] == ' ';
        if (!fg_any(m)) break;
        if (m) --b;
    }
    ok = ok && b - a >= 4 && T[a] == '"';  // KeyMustBeAString; the shortest member is `"":0`
    // "key": up to the next quote, within one 32-bit window of the bitmaps (no loop); a longer key, or a backslash in it
    // (escapes in keys), goes to the exact parser
    const int ks = a + 1;
    int ke = -1;
    if (ok) {
        const uint32_t wq = r5_window(bmQ, ks);
        const int d = fg_ffs(wq) - 1;  // distance of the closing quote
        if (wq != 0u && ks + d < b && (r5_window(bmB, ks) & ((1u << d) - 1u)) == 0u) ke = ks + d;
    }
    ok = ok && ke >= 0;
    int p = ke + 1;
    gf_skip_spaces(T, p, b, ok);
    ok = ok && p < b && T[p] == ':';
    ++p;
    gf_skip_spaces(T, p, b, ok);
    ok = ok && p < b;
    const uint32_t c = ok ? T[p] : 0u;
    name = make_int2(line_off + (ks - ls), ke - ks);
    const uint32_t kbits = ok ? (uint32_t)gf_key_kind(T + ks, ke - ks) << 5 : 0u;  // bits 5..7: the key class, for phase 2
    const bool is_str = ok && c == '"', is_num = ok && (c == '-' || c - '0' <= 9u), is_lit = ok && !is_str && !is_num;
    // string: its closing quote — the first unescaped one — must be the last byte of the member
    const int vs = p + 1;
    int h = vs - 1;
    bool looking = is_str;
    for (;;) {
        if (!fg_any(looking)) break;
        const int hh = gf_next_bit(bmQ, h + 1, b, looking);
        if (looking) {
            h = hh;
            if (h < 0 || !gf_escaped(bmB, h)) looking = false;
        }
    }
    const int ve = h;
    bool str_ok = is_str && h == b - 1;
    bool has_bs = false;
    {   // every backslash of the body starts a valid escape (read.rs parse_escape)
        int pos = vs;
        bool scanning = str_ok;
        for (;;) {
            if (!fg_any(scanning)) break;
            const int x = gf_next_bit(bmB, pos, ve, scanning);
            if (scanning) {
                if (x < 0) {
                    scanning = false;
                } else {
                    has_bs = true;
                    pos = gf_escape_end(T, x, ve);
                    if (pos < 0) { scanning = false; str_ok = false; }
                }
            }
        }
    }
    // true / false / null: the whole token
    bool lit_ok = false;
    uint32_t lit_tag = JT_NULL;
    uint64_t lit_bits = 0;
    if (is_lit) {
        const unsigned long long t8 = lt_load8(T + p);
        const int tl = b - p;
        if (tl == 4 && (uint32_t)t8 == 0x6C6C756Eu) lit_ok = true;                                           // null
        else if (tl == 4 && (uint32_t)t8 == 0x65757274u) { lit_ok = true; lit_tag = JT_BOOL; lit_bits = 1; }  // true
        else if (tl == 5 && (t8 & 0x000000FFFFFFFFFFull) == 0x00000065736C6166ull) { lit_ok = true; lit_tag = JT_BOOL; }  // false
    }
    if (is_str) {
        val = (unsigned long long)(uint32_t)(line_off + (vs - ls)) | ((unsigned long long)(uint32_t)(ve - vs) << 32);
        meta = JT_STRING | (has_bs ? 0x08u : 0u) | kbits;  // FG_EM_UNESCAPE
        return str_ok;
    }
    if (is_num) {
        val = (unsigned long long)(uint32_t)p | ((unsigned long long)(uint32_t)b << 32) | ((unsigned long long)kbits << 48);
        meta = kGfNumber;
        return true;
    }
    val = lit_bits;
    meta = lit_tag | kbits;
    return lit_ok;  // a container as a member value, ExpectedSomeValue, ...: exact parser
}
// the number token left by gf_member (start | end << 32 | key class bits << 48) -> value and tag
FG_DEV bool gf_member_number(const uint8_t* T, unsigned long long span, unsigned long long& val, uint32_t& meta) {
    const uint32_t kbits = (uint32_t)(span >> 48);
    Json j;
    j.p = T;
    j.len = (int)((span >> 32) & 0xFFFFu);
    j.i = (int)(uint32_t)(span & 0xFFFFu);
    j.mode2 = false;
    uint32_t tag = JT_NULL;
    uint64_t bits = 0;
    bool ok;
    if (T[j.i] == '-') {
        ++j.i;
        ok = json_number(j, false, tag, bits);
    } else {
        ok = json_number(j, true, tag, bits);
    }
    if (!ok || j.i != j.len) return false;
    val = bits;
    meta = tag | kbits;
    return true;
}

// Phase 2 for members produced by gf_member (raw keys, key class in bits 5..7 of meta): BTreeMap order = stable insertion
// sort of an index permutation — by the 8-byte key prefix, the bytes only when two prefixes tie —, the last duplicate wins,
// then the rule of the key class.  Same result as gelf_finish_local (fg_gelf.cuh) on the same members.
FG_DEV void gf_finish(bytes_t p, int line_off, const Members& M, LineResult& r, GelfAcc& g, const EntrySink& sink, uint32_t sbase) {
    const uint32_t m = M.m;
    unsigned long long pre[kMaxLocalMembers];
    uint8_t ord[kMaxLocalMembers];
    for (uint32_t a = 0; a < m; ++a) pre[a] = gf_key_prefix(p + (M.name[a].x - line_off), M.name[a].y);
    auto cmp = [&](uint32_t x, uint32_t y) {  // key x vs key y
        if (pre[x] != pre[y]) return pre[x] < pre[y] ? -1 : 1;
        const int2 a = M.name[x], b = M.name[y];
        if (a.y <= 8 && b.y <= 8) return 0;  // both keys are their prefix
        return raw_key_cmp(p, a.x - line_off, a.x - line_off + a.y, b.x - line_off, b.x - line_off + b.y);
    };
    for (uint32_t a = 0; a < m; ++a) {
        int b = (int)a - 1;
        while (b >= 0 && cmp(ord[b], a) > 0) {
            ord[b + 1] = ord[b];
            --b;
        }
        ord[b + 1] = (uint8_t)a;
    }
    uint32_t gi = 0;
    while (gi < m && g.status == FG_ST_OK) {
        uint32_t ge = gi + 1;  // group of equal keys [gi, ge): the last inserted value wins
        while (ge < m && cmp(ord[gi], ord[ge]) == 0) ++ge;
        const uint32_t w = ord[ge - 1];
        gelf_apply_kind((int)(M.meta[w] >> 5), p, line_off, false, M.name[w], M.val[w], M.meta[w] & 0x0Fu, r, g, sink, sbase);
        gi = ge;
    }
}

}  // namespace fg
