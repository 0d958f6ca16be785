// fg_gelf.cuh — one GELF (JSON) line -> Record fields, on device.
//
// H100-native replacement for GelfDecoder::decode
// (flowgger src/flowgger/decoder/gelf_decoder.rs:34-125).  The JSON semantics are those of the
// un-vendored serde_json ~0.8 the reference links (Cargo.toml:51), restated from its published source:
//   de.rs   parse_value / parse_integer / parse_long_integer / parse_number / parse_decimal /
//           parse_exponent / parse_exponent_overflow / visit_f64_from_parts, MapVisitor / SeqVisitor
//   read.rs parse_str_bytes / parse_escape / decode_hex_escape
//   value.rs Value::{Null,Bool,I64,U64,F64,String,Array,Object}, object = BTreeMap<String, Value>
// i.e. byte-lexicographic iteration over the UNESCAPED keys, last duplicate wins, integers are
// U64 / I64 (negative only) / F64 (overflow), floats are significand(u64) */ 10^k (not correctly rounded).
//
// Phase 1 validates the whole document and stores the top-level members, in document order, as
// provisional rows of the side table; phase 2 sorts them by unescaped key, keeps the last duplicate
// and applies the reference's per-key rules in that order, so the first error in SORTED order wins.
#pragma once
#include "fg_common.cuh"
#include "fg_float.cuh"
#include "fg_rfc5424.cuh"
#include "fg_status.h"

namespace fg {

enum : uint32_t { JT_STRING = 0, JT_BOOL = 1, JT_F64 = 2, JT_I64 = 3, JT_U64 = 4, JT_NULL = 5, JT_CONTAINER = 6 };
enum : int { JS_OK = 0, JS_SYNTAX = 1, JS_CONTROL = 2 };  // JS_CONTROL == ErrorCode::InvalidUnicodeCodePoint

struct Json {
    bytes_t p;
    int len;
    int i;
    bool mode2;  // parsing `line.replace('\n', "\\n")` (gelf_decoder.rs:44-46) without materialising it
};

FG_DEV void json_ws(Json& j) {  // parse_whitespace: ' ' '\n' '\t' '\r'
    while (j.i < j.len) {
        const uint32_t c = j.p[j.i];
        // in the retry text every LF has become the two bytes `\n`, which is not whitespace
        if (c == ' ' || c == '\t' || c == '\r' || (c == '\n' && !j.mode2)) ++j.i;
        else break;
    }
}

FG_DEV bool json_hex4(Json& j, uint32_t& n) {
    if (j.i + 4 > j.len) return false;
    n = 0;
    for (int k = 0; k < 4; ++k) {
        const uint32_t c = j.p[j.i + k];
        uint32_t v;
        if (c - '0' <= 9u) v = c - '0';
        else if ((c | 0x20u) - 'a' <= 5u) v = (c | 0x20u) - 'a' + 10u;
        else return false;
        n = n * 16u + v;
    }
    j.i += 4;
    return true;
}

// read.rs parse_str_bytes; j.i is just past the opening quote.  On JS_OK: [s,e) is the raw body, j.i past the closing quote.
static __device__ __noinline__ int json_string(Json& j, int& s, int& e, bool& has_bs) {
    s = j.i;
    has_bs = false;
    const uint32_t b0 = (uint32_t)(size_t)j.p & 15u;
    const uint4* qp = (const uint4*)(j.p - b0);
    for (;;) {
        if (j.i >= j.len) return JS_SYNTAX;  // EOFWhileParsingString
        {
            // 16 bytes per step up to the next '"', '\\' or control byte (read.rs ESCAPE table)
            bool hit;
            j.i = scan_block16_json(qp, b0, j.i, hit);
            if (!hit) continue;
            if (j.i >= j.len) return JS_SYNTAX;  // the hit lies past the end of the line
        }
        const uint32_t c = j.p[j.i];
        if (c == '"') {
            e = j.i;
            ++j.i;
            return JS_OK;
        }
        if (c == '\\') {
            has_bs = true;
            ++j.i;
            if (j.i >= j.len) return JS_SYNTAX;
            const uint32_t x = j.p[j.i++];
            switch (x) {
                case '"': case '\\': case '/': case 'b': case 'f': case 'n': case 'r': case 't': break;
                case 'u': {
                    uint32_t n1;
                    if (!json_hex4(j, n1)) return JS_SYNTAX;
                    if (n1 >= 0xDC00u && n1 <= 0xDFFFu) return JS_SYNTAX;  // LoneLeadingSurrogateInHexEscape
                    if (n1 >= 0xD800u && n1 <= 0xDBFFu) {
                        if (j.i + 2 > j.len) return JS_SYNTAX;
                        if (j.p[j.i] != '\\' || j.p[j.i + 1] != 'u') return JS_SYNTAX;
                        j.i += 2;
                        uint32_t n2;
                        if (!json_hex4(j, n2)) return JS_SYNTAX;
                        if (n2 < 0xDC00u || n2 > 0xDFFFu) return JS_SYNTAX;
                    }
                    break;
                }
                case '\n':
                    // retry text: `\` + LF became `\\` + `n`: a valid escape followed by a plain 'n'
                    if (!j.mode2) return JS_SYNTAX;
                    break;
                default: return JS_SYNTAX;  // InvalidEscape
            }
            continue;
        }
        // control byte (< 0x20)
        if (!j.mode2) return JS_CONTROL;  // first parse: InvalidUnicodeCodePoint -> the caller retries
        if (c != '\n') return JS_SYNTAX;  // retry text still holds this control byte
        ++j.i;
    }
}

// de.rs number parsing.  j.i at the first byte after an optional '-'.  tag/bits receive the Value.
static __device__ __noinline__ bool json_number(Json& j, bool pos, uint32_t& tag, uint64_t& bits) {
    // parse_integer
    if (j.i >= j.len) return false;
    uint32_t c = j.p[j.i++];
    uint64_t sig = 0;
    int exp10 = 0;
    bool long_int = false;
    if (c == '0') {
        if (j.i < j.len && (uint32_t)j.p[j.i] - '0' <= 9u) return false;  // leading zero
    } else if (c - '1' <= 8u) {
        sig = c - '0';
        while (j.i < j.len) {
            const uint32_t d = (uint32_t)j.p[j.i] - '0';
            if (d > 9u) break;
            ++j.i;
            if (sig >= 1844674407370955161ull && (sig > 1844674407370955161ull || d > 5u)) {  // overflow!(sig*10+d, u64::MAX)
                long_int = true;
                exp10 = 1;
                break;
            }
            sig = sig * 10ull + d;
        }
    } else {
        return false;
    }
    bool is_float = long_int;
    if (long_int) {  // parse_long_integer: further integer digits only scale
        while (j.i < j.len && (uint32_t)j.p[j.i] - '0' <= 9u) { ++j.i; ++exp10; }
    }
    c = j.i < j.len ? j.p[j.i] : 0u;
    if (c == '.') {  // parse_decimal
        is_float = true;
        ++j.i;
        bool at_least_one = false;
        while (j.i < j.len) {
            const uint32_t d = (uint32_t)j.p[j.i] - '0';
            if (d > 9u) break;
            ++j.i;
            at_least_one = true;
            if (sig >= 1844674407370955161ull && (sig > 1844674407370955161ull || d > 5u)) {
                while (j.i < j.len && (uint32_t)j.p[j.i] - '0' <= 9u) ++j.i;
                break;
            }
            sig = sig * 10ull + d;
            --exp10;
        }
        if (!at_least_one) return false;
        c = j.i < j.len ? j.p[j.i] : 0u;
    }
    if (c == 'e' || c == 'E') {  // parse_exponent
        is_float = true;
        ++j.i;
        bool pos_exp = true;
        if (j.i < j.len && j.p[j.i] == '+') ++j.i;
        else if (j.i < j.len && j.p[j.i] == '-') { pos_exp = false; ++j.i; }
        if (j.i >= j.len) return false;
        uint32_t d = (uint32_t)j.p[j.i++] - '0';
        if (d > 9u) return false;
        int ex = (int)d;
        bool overflow = false;
        while (j.i < j.len) {
            d = (uint32_t)j.p[j.i] - '0';
            if (d > 9u) break;
            ++j.i;
            if (ex >= 214748364 && (ex > 214748364 || d > 7u)) {  // overflow!(ex*10+d, i32::MAX)
                overflow = true;
                break;
            }
            ex = ex * 10 + (int)d;
        }
        if (overflow) {  // parse_exponent_overflow
            if (sig != 0 && pos_exp) return false;  // NumberOutOfRange
            while (j.i < j.len && (uint32_t)j.p[j.i] - '0' <= 9u) ++j.i;
            tag = JT_F64;
            bits = pos ? 0ull : 0x8000000000000000ull;
            return true;
        }
        long long fe = pos_exp ? (long long)exp10 + ex : (long long)exp10 - ex;  // saturating_add / saturating_sub
        if (fe > 2147483647LL) fe = 2147483647LL;
        if (fe < -2147483648LL) fe = -2147483648LL;
        exp10 = (int)fe;
    }
    if (is_float) {
        double f;
        // exponent == i32::MIN: |exponent| is not a table index either (release-mode wrap), same path as "too large"
        if (!serde_f64_from_parts(pos, sig, exp10, f)) return false;
        tag = JT_F64;
        bits = (uint64_t)__double_as_longlong(f);
        return true;
    }
    if (pos) {
        tag = JT_U64;
        bits = sig;
    } else {
        const long long neg = (long long)(0ull - sig);  // (sig as i64).wrapping_neg()
        if (neg > 0) {
            tag = JT_F64;
            bits = (uint64_t)__double_as_longlong(-__ull2double_rn(sig));
        } else if (neg < 0) {
            tag = JT_I64;
            bits = (uint64_t)neg;
        } else {
            tag = JT_U64;  // Value visitor: visit_i64(0) -> U64(0)
            bits = 0;
        }
    }
    return true;
}

FG_DEV bool json_lit(Json& j, const char* rest, int n) {  // parse_ident
    if (j.i + n > j.len) return false;
    for (int k = 0; k < n; ++k)
        if (j.p[j.i + k] != (uint8_t)rest[k]) return false;
    j.i += n;
    return true;
}

// Iterates the UNESCAPED bytes of a validated JSON string body.
struct KeyIter {
    bytes_t p;
    int i, end;
    bool mode2;
    uint32_t pend;  // queued bytes (low byte first)
    int npend;
};
FG_DEV void key_iter_init(KeyIter& k, bytes_t p, int a, int b, bool mode2) {
    k.p = p; k.i = a; k.end = b; k.mode2 = mode2; k.pend = 0; k.npend = 0;
}
static __device__ __noinline__ int key_iter_next(KeyIter& k) {  // -1 at the end
    if (k.npend) {
        const int b = (int)(k.pend & 0xFFu);
        k.pend >>= 8;
        --k.npend;
        return b;
    }
    if (k.i >= k.end) return -1;
    uint32_t c = k.p[k.i++];
    if (c != '\\') return (int)c;
    const uint32_t x = k.p[k.i++];
    switch (x) {
        case 'b': return 0x08;
        case 'f': return 0x0C;
        case 'n': return 0x0A;
        case 'r': return 0x0D;
        case 't': return 0x09;
        case '\n': k.pend = 'n'; k.npend = 1; return '\\';  // retry text: `\\` then 'n'
        case 'u': {
            uint32_t n = 0;
            for (int q = 0; q < 4; ++q) {
                const uint32_t h = k.p[k.i + q];
                n = n * 16u + (h - '0' <= 9u ? h - '0' : (h | 0x20u) - 'a' + 10u);
            }
            k.i += 4;
            if (n >= 0xD800u && n <= 0xDBFFu) {
                uint32_t n2 = 0;
                for (int q = 0; q < 4; ++q) {
                    const uint32_t h = k.p[k.i + 2 + q];
                    n2 = n2 * 16u + (h - '0' <= 9u ? h - '0' : (h | 0x20u) - 'a' + 10u);
                }
                k.i += 6;
                n = (((n - 0xD800u) << 10) | (n2 - 0xDC00u)) + 0x10000u;
            }
            if (n < 0x80u) return (int)n;
            if (n < 0x800u) { k.pend = 0x80u | (n & 0x3Fu); k.npend = 1; return (int)(0xC0u | (n >> 6)); }
            if (n < 0x10000u) {
                k.pend = (0x80u | ((n >> 6) & 0x3Fu)) | ((0x80u | (n & 0x3Fu)) << 8);
                k.npend = 2;
                return (int)(0xE0u | (n >> 12));
            }
            k.pend = (0x80u | ((n >> 12) & 0x3Fu)) | ((0x80u | ((n >> 6) & 0x3Fu)) << 8) | ((0x80u | (n & 0x3Fu)) << 16);
            k.npend = 3;
            return (int)(0xF0u | (n >> 18));
        }
        default: return (int)x;  // '"' '\\' '/'
    }
}
// String Ord when neither key holds an escape: plain byte-wise compare of the raw spans (the common case)
FG_DEV int raw_key_cmp(bytes_t p, int a0, int a1, int b0, int b1) {
    const int la = a1 - a0, lb = b1 - b0, n = la < lb ? la : lb;
    for (int k = 0; k < n; ++k) {
        const int ca = p[a0 + k], cb = p[b0 + k];
        if (ca != cb) return ca < cb ? -1 : 1;
    }
    return la == lb ? 0 : (la < lb ? -1 : 1);
}
FG_DEV bool raw_str_is(bytes_t p, int a0, int a1, const char* lit, int n) {
    if (a1 - a0 != n) return false;
    for (int k = 0; k < n; ++k)
        if (p[a0 + k] != (uint8_t)lit[k]) return false;
    return true;
}

// String Ord on the unescaped bytes
static __device__ __noinline__ int json_key_cmp(bytes_t p, int a0, int a1, int b0, int b1, bool mode2) {
    KeyIter x, y;
    key_iter_init(x, p, a0, a1, mode2);
    key_iter_init(y, p, b0, b1, mode2);
    for (;;) {
        const int cx = key_iter_next(x), cy = key_iter_next(y);
        if (cx != cy) return cx < cy ? -1 : 1;
        if (cx < 0) return 0;
    }
}
static __device__ __noinline__ bool json_str_is(bytes_t p, int a0, int a1, bool mode2, const char* lit, int n) {
    KeyIter x;
    key_iter_init(x, p, a0, a1, mode2);
    for (int k = 0; k < n; ++k)
        if (key_iter_next(x) != (int)(uint8_t)lit[k]) return false;
    return key_iter_next(x) < 0;
}

// serde_json 0.8 ser.rs escape_bytes: `"` `\` \b \f \n \r \t get a backslash form (returns the second byte), else 0
FG_DEV uint32_t json_escape_of(uint32_t c) {
    if (c == '"' || c == '\\') return c;
    if (c >= 0x20u) return 0u;
    return c == 8u ? 'b' : c == 9u ? 't' : c == 10u ? 'n' : c == 12u ? 'f' : c == 13u ? 'r' : 0u;
}

// One step of re-encoding a validated JSON string body p[i, end) as the text serde_json prints for its unescaped bytes
// (GelfDecoder::decode unescapes, GelfEncoder::encode escapes again): the source escape — or raw byte — at p[i] becomes
// 1..4 output bytes in w (low byte first), i moves past it; returns the byte count.  The unescape is KeyIter's and the
// escape json_escape_of, so decoder and encoder cannot disagree on what a string holds.  At most 4 bytes: a \uXXXX
// gives 1..3 bytes of UTF-8 (a byte below 0x80 escaped to 2 at most), a surrogate pair 4, `\` + LF of a retry line
// the 3 bytes `\\n`.
FG_DEV int json_transcode_step(bytes_t p, int& i, int end, bool mode2, uint32_t& w) {
    KeyIter it;
    key_iter_init(it, p, i, end, mode2);
    w = 0;
    int n = 0;
    do {
        const uint32_t c = (uint32_t)key_iter_next(it);
        const uint32_t e = json_escape_of(c);
        w |= (e ? ('\\' | (e << 8)) : c) << (8 * n);
        n += e ? 2 : 1;
    } while (it.npend);
    i = it.i;
    return n;
}


// One step of reading a validated JSON string body p[i, end) as its unescaped bytes (the LTSV encoder writes the text,
// not JSON): the source escape — or raw byte — at p[i] becomes 1..4 bytes in w (low byte first), i moves past it;
// returns the byte count.  At most 4: a surrogate pair is 4 bytes of UTF-8, `\` + LF of a retry line `\` and 'n'.
FG_DEV int json_unescape_step(bytes_t p, int& i, int end, bool mode2, uint32_t& w) {
    KeyIter it;
    key_iter_init(it, p, i, end, mode2);
    w = 0;
    int n = 0;
    do {
        w |= (uint32_t)key_iter_next(it) << (8 * n);
        ++n;
    } while (it.npend);
    i = it.i;
    return n;
}

// Top-level members of one line while it is being parsed: the first kMaxLocalMembers live in per-thread local
// memory (L1-resident); an object with more members spills everything to the scratch table (rare).
constexpr int kMaxLocalMembers = 24;
struct Members {
    int2 name[kMaxLocalMembers];
    unsigned long long val[kMaxLocalMembers];
    uint8_t meta[kMaxLocalMembers];
    uint32_t m;
    bool spilled;
};
FG_DEV void members_put(Members& M, const EntrySink& sink, uint32_t sbase, int2 name, unsigned long long val, uint32_t meta) {
    if (!M.spilled && M.m < (uint32_t)kMaxLocalMembers) {
        M.name[M.m] = name;
        M.val[M.m] = val;
        M.meta[M.m] = (uint8_t)meta;
    } else {
        if (!M.spilled) {
            for (uint32_t k = 0; k < M.m; ++k) {
                sink.name[sbase + k] = M.name[k];
                sink.val[sbase + k] = M.val[k];
                sink.meta[sbase + k] = M.meta[k];
            }
            M.spilled = true;
        }
        sink.name[sbase + M.m] = name;
        sink.val[sbase + M.m] = val;
        sink.meta[sbase + M.m] = (uint8_t)meta;
    }
    ++M.m;
}

// One full parse of the document in the given mode.  Returns JS_*; on JS_OK `is_object` tells whether the
// top-level value is an object and `m` members were staged at sink[sbase ..) in document order.
static __device__ __noinline__ int gelf_parse_document(bytes_t p, int len, int line_off, uint32_t sbase, bool mode2,
                                                const EntrySink& sink, bool& is_object, Members& M) {
    Json j;
    j.p = p; j.len = len; j.i = 0; j.mode2 = mode2;
    uint32_t stack[4] = {0u, 0u, 0u, 0u};  // bit d-1: container at depth d is an object
    int depth = 0;                          // open containers (serde: remaining_depth = 128 - depth)
    M.m = 0;
    M.spilled = false;
    is_object = false;
    // member being built (only meaningful at depth 1 of a top-level object)
    int key_s = 0, key_e = 0;
    bool key_bs = false;
    enum { ST_VALUE, ST_AFTER, ST_KEY } st = ST_VALUE;
    for (;;) {
        if (st == ST_VALUE) {
            json_ws(j);
            if (j.i >= j.len) return JS_SYNTAX;  // EOFWhileParsingValue
            const uint32_t c = j.p[j.i];
            uint32_t tag = JT_NULL;
            uint64_t bits = 0;
            uint32_t vflags = 0;
            bool scalar = true;
            if (c == '"') {
                ++j.i;
                int s, e;
                bool bs;
                const int rc = json_string(j, s, e, bs);
                if (rc != JS_OK) return rc;
                tag = JT_STRING;
                bits = (uint64_t)(uint32_t)(line_off + s) | ((uint64_t)(uint32_t)(e - s) << 32);
                vflags = bs ? 0x08u : 0u;  // FG_EM_UNESCAPE
            } else if (c == '-') {
                ++j.i;
                if (!json_number(j, false, tag, bits)) return JS_SYNTAX;
            } else if (c - '0' <= 9u) {
                if (!json_number(j, true, tag, bits)) return JS_SYNTAX;
            } else if (c == 'n') {
                ++j.i;
                if (!json_lit(j, "ull", 3)) return JS_SYNTAX;
                tag = JT_NULL;
            } else if (c == 't') {
                ++j.i;
                if (!json_lit(j, "rue", 3)) return JS_SYNTAX;
                tag = JT_BOOL;
                bits = 1;
            } else if (c == 'f') {
                ++j.i;
                if (!json_lit(j, "alse", 4)) return JS_SYNTAX;
                tag = JT_BOOL;
                bits = 0;
            } else if (c == '[' || c == '{') {
                if (depth + 1 >= 128) return JS_SYNTAX;  // RecursionLimitExceeded (remaining_depth hits 0)
                ++j.i;
                scalar = false;
                const bool obj = c == '{';
                if (depth == 0) is_object = obj;
                if (depth == 1 && is_object) {  // a container as a top-level member value
                    members_put(M, sink, sbase, make_int2(line_off + key_s, key_e - key_s), 0ull, JT_CONTAINER | (key_bs ? 0x40u : 0u));
                }
                if (obj) stack[depth >> 5] |= 1u << (depth & 31);
                else stack[depth >> 5] &= ~(1u << (depth & 31));
                ++depth;
                json_ws(j);
                if (j.i >= j.len) return JS_SYNTAX;
                const uint32_t c2 = j.p[j.i];
                if (c2 == (obj ? '}' : ']')) {
                    ++j.i;
                    --depth;
                    st = ST_AFTER;
                } else {
                    st = obj ? ST_KEY : ST_VALUE;
                }
            } else {
                return JS_SYNTAX;  // ExpectedSomeValue
            }
            if (scalar) {
                if (depth == 1 && is_object) {
                    members_put(M, sink, sbase, make_int2(line_off + key_s, key_e - key_s), bits, tag | vflags | (key_bs ? 0x40u : 0u));
                }
                st = ST_AFTER;
            }
        } else if (st == ST_KEY) {
            // MapVisitor::visit_key after '{' or ',' : the next token must be a string
            if (j.i >= j.len || j.p[j.i] != '"') return JS_SYNTAX;  // KeyMustBeAString
            ++j.i;
            int s, e;
            bool bs;
            const int rc = json_string(j, s, e, bs);
            if (rc != JS_OK) return rc;
            if (depth == 1) { key_s = s; key_e = e; key_bs = bs; }
            json_ws(j);
            if (j.i >= j.len || j.p[j.i] != ':') return JS_SYNTAX;  // parse_object_colon
            ++j.i;
            st = ST_VALUE;
        } else {  // ST_AFTER: a value just ended
            if (depth == 0) break;
            const bool obj = (stack[(depth - 1) >> 5] >> ((depth - 1) & 31)) & 1u;
            json_ws(j);
            if (j.i >= j.len) return JS_SYNTAX;
            const uint32_t c = j.p[j.i];
            if (c == ',') {
                ++j.i;
                if (obj) { json_ws(j); st = ST_KEY; }
                else st = ST_VALUE;
            } else if (c == (obj ? '}' : ']')) {
                ++j.i;
                --depth;
                st = ST_AFTER;
            } else {
                return JS_SYNTAX;  // ExpectedObjectCommaOrEnd / ExpectedListCommaOrEnd
            }
        }
    }
    json_ws(j);  // Deserializer::end
    if (j.i != j.len) return JS_SYNTAX;  // TrailingCharacters
    return JS_OK;
}

// Per-key rules of gelf_decoder.rs:51-107 applied to one (deduplicated) member, in sorted-key order.
struct GelfAcc {
    uint32_t status, flags, kept;
    bool have_ts;
};
enum { GKEY_OTHER = 0, GKEY_TIMESTAMP, GKEY_HOST, GKEY_SHORT, GKEY_FULL, GKEY_VERSION, GKEY_LEVEL };

// the rule of one key class; `kind` = GKEY_* of the (unescaped) key
FG_DEV void gelf_apply_kind(int kind, bytes_t p, int line_off, bool mode2, int2 name, unsigned long long val, uint32_t meta, LineResult& r,
                            GelfAcc& g, const EntrySink& sink, uint32_t sbase) {
    const int ks = name.x - line_off, ke = ks + name.y;
    const uint32_t tag = meta & 7u;
    const int vs = (int)(uint32_t)(val & 0xFFFFFFFFull) - line_off, vl = (int)(val >> 32);
    const bool kesc = (meta & 0x40u) != 0, vesc = (meta & 0x08u) != 0;
    auto val_is = [&](const char* lit, int n) { return vesc ? json_str_is(p, vs, vs + vl, mode2, lit, n) : raw_str_is(p, vs, vs + vl, lit, n); };
    if (kind == GKEY_TIMESTAMP) {  // as_f64 :53
        if (tag == JT_F64) r.ts = __longlong_as_double((long long)val);
        else if (tag == JT_U64) r.ts = __ull2double_rn(val);
        else if (tag == JT_I64) r.ts = __ll2double_rn((long long)val);
        else g.status = FG_EG_TS;
        g.have_ts = true;
    } else if (kind == GKEY_HOST) {
        if (tag != JT_STRING) g.status = FG_EG_HOST;
        else { r.host_o = vs; r.host_l = vl; if (meta & 0x08u) g.flags |= 0x04u; }
    } else if (kind == GKEY_SHORT) {
        if (tag != JT_STRING) g.status = FG_EG_SHORT;
        else { r.msg_o = vs; r.msg_l = vl; if (meta & 0x08u) g.flags |= 0x08u; }
    } else if (kind == GKEY_FULL) {
        if (tag != JT_STRING) g.status = FG_EG_FULL;
        else { r.full_o = vs; r.full_l = vl; if (meta & 0x08u) g.flags |= 0x10u; }
    } else if (kind == GKEY_VERSION) {
        if (tag != JT_STRING) g.status = FG_EG_VERSION_T;
        else if (!val_is("1.0", 3) && !val_is("1.1", 3)) g.status = FG_EG_VERSION;
    } else if (kind == GKEY_LEVEL) {  // as_u64 :83
        if (tag != JT_U64) g.status = FG_EG_SEV;
        else if (val > 7ull) g.status = FG_EG_SEV_HIGH;
        else r.severity = (uint32_t)val;
    } else {
        if (tag == JT_CONTAINER) g.status = FG_EG_SD_TYPE;  // :97
        else {
            bool under = (ke > ks) && p[ks] == '_';
            if (kesc) {
                KeyIter it;
                key_iter_init(it, p, ks, ke, mode2);
                under = key_iter_next(it) == '_';
            }
            const uint32_t e = sbase + g.kept;
            sink.name[e] = name;
            sink.val[e] = val;
            sink.meta[e] = (uint8_t)((meta & 0x4Fu) | (under ? 0x10u : 0u));  // tag | UNESCAPE | NAME_ESC | NO_PREFIX
            ++g.kept;
        }
    }
}

static __device__ __noinline__ void gelf_apply_member(bytes_t p, int line_off, bool mode2, int2 name, unsigned long long val, uint32_t meta,
                                                      LineResult& r, GelfAcc& g, const EntrySink& sink, uint32_t sbase) {
    const int ks = name.x - line_off, ke = ks + name.y;
    // reserved keys contain no '_' and differ in their first byte: skip the literal compares for ordinary `_extra` keys
    const uint32_t k0 = (ke > ks) ? p[ks] : 0u;
    const bool maybe = k0 == 't' || k0 == 'h' || k0 == 's' || k0 == 'f' || k0 == 'v' || k0 == 'l' || k0 == '\\';
    const bool kesc = (meta & 0x40u) != 0;
    auto key_is = [&](const char* lit, int n) { return kesc ? json_str_is(p, ks, ke, mode2, lit, n) : raw_str_is(p, ks, ke, lit, n); };
    int kind = GKEY_OTHER;
    if (maybe) {
        if (key_is("timestamp", 9)) kind = GKEY_TIMESTAMP;
        else if (key_is("host", 4)) kind = GKEY_HOST;
        else if (key_is("short_message", 13)) kind = GKEY_SHORT;
        else if (key_is("full_message", 12)) kind = GKEY_FULL;
        else if (key_is("version", 7)) kind = GKEY_VERSION;
        else if (key_is("level", 5)) kind = GKEY_LEVEL;
    }
    gelf_apply_kind(kind, p, line_off, mode2, name, val, meta, r, g, sink, sbase);
}

FG_DEV void gelf_result_init(LineResult& r) {
    r.ts = 0.0;
    r.facility = 0xFFu;
    r.severity = 0xFFu;
    r.flags = 0;
    r.host_o = r.app_o = r.proc_o = r.mid_o = r.msg_o = r.full_o = -1;
    r.host_l = r.app_l = r.proc_l = r.mid_l = r.msg_l = r.full_l = 0;
    r.n_entries = 0;
    r.status = FG_EG_JSON;
}

// Phase 2 over members held in local memory: BTreeMap order = stable insertion sort of an index permutation by unescaped
// key, the last duplicate wins, then the per-key rules in that order (rows go to sink[sbase ..)).
FG_DEV void gelf_finish_local(bytes_t p, int line_off, bool mode2, const Members& M, LineResult& r, GelfAcc& g, const EntrySink& sink,
                              uint32_t sbase) {
    const uint32_t m = M.m;
    uint8_t ord[kMaxLocalMembers];
    for (uint32_t a = 0; a < m; ++a) {
        const int2 kn = M.name[a];
        int b = (int)a - 1;
        const bool kn_esc = (M.meta[a] & 0x40u) != 0;
        while (b >= 0) {
            const int2 on = M.name[ord[b]];
            const int cmp = (kn_esc || (M.meta[ord[b]] & 0x40u))
                                ? json_key_cmp(p, on.x - line_off, on.x - line_off + on.y, kn.x - line_off, kn.x - line_off + kn.y, mode2)
                                : raw_key_cmp(p, on.x - line_off, on.x - line_off + on.y, kn.x - line_off, kn.x - line_off + kn.y);
            if (cmp <= 0) break;
            ord[b + 1] = ord[b];
            --b;
        }
        ord[b + 1] = (uint8_t)a;
    }
    uint32_t gi = 0;
    while (gi < m && g.status == FG_ST_OK) {
        uint32_t ge = gi + 1;  // group of equal keys [gi, ge): the last inserted value wins
        const int2 gn = M.name[ord[gi]];
        const int ks = gn.x - line_off, ke = ks + gn.y;
        const bool g_esc = (M.meta[ord[gi]] & 0x40u) != 0;
        while (ge < m) {
            const int2 nn = M.name[ord[ge]];
            const int cmp = (g_esc || (M.meta[ord[ge]] & 0x40u)) ? json_key_cmp(p, ks, ke, nn.x - line_off, nn.x - line_off + nn.y, mode2)
                                                                : raw_key_cmp(p, ks, ke, nn.x - line_off, nn.x - line_off + nn.y);
            if (cmp != 0) break;
            ++ge;
        }
        const uint32_t w = ord[ge - 1];
        gelf_apply_member(p, line_off, mode2, M.name[w], M.val[w], M.meta[w], r, g, sink, sbase);
        gi = ge;
    }
}

// gelf_decoder.rs:109-110 and the shape of an error row
FG_DEV void gelf_finalize(LineResult& r, GelfAcc& g) {
    if (g.status == FG_ST_OK) {
        if (r.host_o < 0) g.status = FG_EG_MISSING_HOST;  // :110
        else if (!g.have_ts) g.flags |= 0x01u;            // FG_FLAG_TS_MISSING :109
    }
    if (g.status == FG_ST_OK) r.n_entries = g.kept;
    else { r.host_o = r.msg_o = r.full_o = -1; r.severity = 0xFFu; r.ts = 0.0; }
    r.flags = g.flags;
    r.status = g.status;
}

// All 32 lanes call this; idle lanes pass active_line = false.
FG_DEV void gelf_parse_line(bytes_t p, int len, int line_off, uint32_t sbase, bool active_line, LineResult& r,
                            const EntrySink& sink) {
    gelf_result_init(r);
    if (active_line) {
        GelfAcc g;
        g.status = FG_ST_OK;
        g.flags = 0;
        g.kept = 0;
        g.have_ts = false;
        Members M;
        bool is_object = false, mode2 = false;
        int rc = gelf_parse_document(p, len, line_off, sbase, false, sink, is_object, M);
        if (rc == JS_CONTROL) {  // gelf_decoder.rs:44-46
            mode2 = true;
            g.flags |= 0x20u;  // FG_FLAG_NL_RETRY
            rc = gelf_parse_document(p, len, line_off, sbase, true, sink, is_object, M);
        }
        if (rc != JS_OK) g.status = FG_EG_JSON;        // :49
        else if (!is_object) g.status = FG_EG_EMPTY;   // :50
        const uint32_t m = M.m;
        if (g.status == FG_ST_OK && !M.spilled) {
            gelf_finish_local(p, line_off, mode2, M, r, g, sink, sbase);
        } else if (g.status == FG_ST_OK) {
            // > kMaxLocalMembers members: same algorithm in place on the scratch table
            for (uint32_t a = 1; a < m; ++a) {
                const int2 kn = sink.name[sbase + a];
                const unsigned long long kv = sink.val[sbase + a];
                const uint8_t km = sink.meta[sbase + a];
                int b = (int)a - 1;
                while (b >= 0) {
                    const int2 on = sink.name[sbase + b];
                    if (json_key_cmp(p, on.x - line_off, on.x - line_off + on.y, kn.x - line_off, kn.x - line_off + kn.y, mode2) <= 0) break;
                    sink.name[sbase + b + 1] = on;
                    sink.val[sbase + b + 1] = sink.val[sbase + b];
                    sink.meta[sbase + b + 1] = sink.meta[sbase + b];
                    --b;
                }
                if (b + 1 != (int)a) {
                    sink.name[sbase + b + 1] = kn;
                    sink.val[sbase + b + 1] = kv;
                    sink.meta[sbase + b + 1] = km;
                }
            }
            uint32_t gi = 0;
            while (gi < m && g.status == FG_ST_OK) {
                uint32_t ge = gi + 1;
                const int2 gn = sink.name[sbase + gi];
                const int ks = gn.x - line_off, ke = ks + gn.y;
                while (ge < m) {
                    const int2 nn = sink.name[sbase + ge];
                    if (json_key_cmp(p, ks, ke, nn.x - line_off, nn.x - line_off + nn.y, mode2) != 0) break;
                    ++ge;
                }
                // rows [0, kept) are rewritten in place: kept <= gi, so nothing unread is clobbered
                gelf_apply_member(p, line_off, mode2, sink.name[sbase + ge - 1], sink.val[sbase + ge - 1], sink.meta[sbase + ge - 1], r, g,
                                  sink, sbase);
                gi = ge;
            }
        }
        gelf_finalize(r, g);
    }
    __syncwarp();
}

}  // namespace fg
