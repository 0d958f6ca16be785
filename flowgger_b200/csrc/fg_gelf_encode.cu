// fg_gelf_encode.cu — the stage AFTER the decoder, fused on the device: Record -> GELF JSON bytes (SURVEY.md §8(f) N2).
//
// H100-native replacement for GelfEncoder::encode (flowgger src/flowgger/encoder/gelf_encoder.rs:59-115), which
// every splitter calls right after Decoder::decode (splitter/line_splitter.rs:50-52).  The JSON text is what
// serde_json "~0.8" `to_vec` prints for the BTreeMap the reference builds: keys in byte order, a later insert replaces
// an earlier one (SD pairs replace fixed fields, output.gelf_extra replaces everything), compact separators, strings
// with `"` `\\` \b \f \n \r \t escaped, Record.ts through dtoa (fg_dtoa.cuh).
//
// Input = the decoder's device-resident results; nothing of them travels to the host in this mode.  Three record
// sources, chosen at compile time (the kernels are templates on the source, everything after the record view is shared):
//   From5424  compact rows + 8-byte entries + arena, or wide rows (structured data; every fixed field present)
//   From3164  the row columns of parse3164_kernel + the arena of re-joined messages (rfc3164_decoder.rs:71-82, 106-117:
//             no appname, procid or structured data; no severity without <PRI>; msg always Some, possibly "")
//   FromLtsv  the row columns of parse_ltsv_kernel + its 17-byte side table (ltsv_decoder.rs:87-221: no appname, procid
//             or sd_id; no severity without `level`; msg None without `message`).  A pair's key is '_' + name + the
//             type's suffix (FG_EM_SUFFIX), so keys are ordered and de-duplicated on that composed text; a typed value
//             (bool, f64, i64, u64) is written as JSON, not as its source text.
// Launches per chunk of lines:
//   gelf_size_kernel   one thread per line: exact length of its record (0 for a line the decoder rejected); the bytes of
//                      the CTA's 256 lines are staged in shared memory by one TMA bulk copy and handed to the threads
//                      in order of line length (both kernels)
//   cub exclusive sum  record offsets inside the chunk
//   gelf_write_kernel  one thread per line writes its record; output bytes are assembled four at a time and stored as
//                      aligned 32-bit words, so a record costs a quarter of the store instructions / L2 requests of a
//                      byte-wise copy
// Both kernels run ONE emit routine over a counting or a writing sink, so the two passes cannot disagree.
// All SD names start with '_' (rfc5424_decoder.rs:221), i.e. they sort before every fixed GELF key; the general merge
// with the pre-sorted static items (fixed keys + extras, prepared on the host once) still compares full keys.
#include <cub/device/device_scan.cuh>

#include "fg_kernels.cuh"

#include "fg_common.cuh"
#include "fg_dtoa.cuh"
#include "fg_r5fast.cuh"
#include "fg_status.h"
#include "fg_tma.cuh"

namespace fg {

namespace {

struct Span {
    const uint8_t* p;
    int len;
};

// record lengths are 64-bit all the way to the output offsets: one record, or one launch's records, may pass 4 GiB
struct CountSink {
    unsigned long long n = 0;
    __device__ __forceinline__ void push(uint32_t, int k) { n += (unsigned)k; }
    __device__ __forceinline__ void finish() {}
};
// bytes -> aligned 32-bit stores: a 64-bit shift register takes 1 or 4 bytes per push (the same instructions for both, so
// lanes that push one byte and lanes that push four stay together) and gives up a word whenever it holds four; only the
// up-to-three bytes in front of the first aligned address and the tail of the record are stored byte-wise
struct WordSink {
    uint8_t* p;
    unsigned long long acc = 0;  // pending bytes, low byte first
    int nacc = 0;                // 0..3 between calls
    int head;                    // bytes still to store singly before p is 4-byte aligned
    __device__ __forceinline__ explicit WordSink(uint8_t* at) : p(at), head((int)((4u - ((uint32_t)(size_t)at & 3u)) & 3u)) {}
    // k = 1 or 4 bytes of w, low byte first (unused high bytes of w are 0)
    __device__ __forceinline__ void push(uint32_t w, int k) {
        if (head) {  // the first one or two pushes of a record
            while (head && k) {
                *p++ = (uint8_t)w;
                w >>= 8;
                --head;
                --k;
            }
            if (k == 0) return;
        }
        acc |= (unsigned long long)w << (8 * nacc);
        nacc += k;
        if (nacc >= 4) {
            *reinterpret_cast<uint32_t*>(p) = (uint32_t)acc;
            p += 4;
            acc >>= 32;
            nacc -= 4;
        }
    }
    __device__ __forceinline__ void finish() {
        for (int k = 0; k < nacc; ++k) p[k] = (uint8_t)(acc >> (8 * k));
        nacc = 0;
    }
};

// An LTSV record's sink: the extent of the side table's value column, which tells run_segments the number segments
template <class Sink>
struct NumSink {
    Sink& s;
    const unsigned long long* vals;
    uint32_t cap;
    __device__ __forceinline__ void push(uint32_t w, int k) { s.push(w, k); }
};

// byte-order comparison of ('_' + a) with b
__device__ __forceinline__ int cmp_sd_key(Span a, Span b) {
    if (b.len == 0) return 1;
    if ((uint32_t)'_' != b.p[0]) return (uint32_t)'_' < b.p[0] ? -1 : 1;
    const int n = min(a.len, b.len - 1);
    for (int k = 0; k < n; ++k) {
        const uint32_t x = a.p[k], y = b.p[k + 1];
        if (x != y) return x < y ? -1 : 1;
    }
    return a.len == b.len - 1 ? 0 : (a.len < b.len - 1 ? -1 : 1);
}
__device__ __forceinline__ int cmp_names(Span a, Span b) {
    const int n = min(a.len, b.len);
    for (int k = 0; k < n; ++k) {
        const uint32_t x = a.p[k], y = b.p[k];
        if (x != y) return x < y ? -1 : 1;
    }
    return a.len == b.len ? 0 : (a.len < b.len ? -1 : 1);
}

// One decoded line, whichever table it lives in
struct RecView {
    bool ok;
    bool wide;
    double ts;
    uint32_t severity;
    Span host, app, proc, msg, full;  // msg.p == nullptr: None
    Span sd_id;                        // id of the LAST element (gelf_encoder.rs:97-99 inserts "sd_id" per element)
    bool has_sd;
    uint32_t first, count;             // entries8 range, or wide-entry range
    const uint8_t* line;
};

// `src` = where the bytes of the caller's buffer are read from: the staged tile (src[k] = byte base + k) or global memory
// (base = 0).  Spans of the compact rows are relative to the line, wide rows carry absolute spans.
struct ByteSource {
    const uint8_t* p;  // p[abs - base] is byte `abs`
    int base;
    __device__ __forceinline__ const uint8_t* at(int abs) const { return p + (abs - base); }
};

__device__ __forceinline__ void load_view(const GelfEncodeParams& P, const ByteSource& B, int i, RecView& r) {
    const uint4 lo4 = P.rows[2 * (size_t)i], hi4 = P.rows[2 * (size_t)i + 1];
    const uint32_t meta = lo4.z;
    r.ok = (meta & 0xFFu) == 0u;
    r.wide = ((meta >> 24) & kFlagWide) != 0u;
    r.has_sd = false;
    r.sd_id = Span{nullptr, 0};
    r.msg = Span{nullptr, 0};
    r.first = r.count = 0;
    if (!r.ok) return;
    r.severity = (meta >> 16) & 0xFFu;
    const int o0 = P.offsets[i];
    r.line = B.at(o0);
    if (r.wide) {
        if (lo4.w >= P.wide_cap) { r.ok = false; return; }
        const WideRow& w = P.wide_rows[lo4.w];
        r.ts = w.ts;
        r.host = Span{B.at(w.host.x), w.host.y};
        r.app = Span{B.at(w.app.x), w.app.y};
        r.proc = Span{B.at(w.proc.x), w.proc.y};
        if (w.msg.x >= 0) r.msg = Span{B.at(w.msg.x), w.msg.y};
        r.full = Span{B.at(max(w.full.x, o0)), w.full.x >= 0 ? w.full.y : 0};
        r.first = (uint32_t)w.sd.x;
        r.count = (uint32_t)w.sd.y;
        if ((unsigned long long)r.first + r.count > (unsigned long long)P.wentry_cap) { r.ok = false; return; }
        for (uint32_t e = r.first; e < r.first + r.count; ++e)
            if ((P.wentry_meta[e] & 0x07u) == 7u) {
                r.has_sd = true;
                r.sd_id = Span{B.at(P.wentry_name[e].x), P.wentry_name[e].y};
            }
        return;
    }
    r.ts = __hiloint2double((int)lo4.y, (int)lo4.x);
    const int sp1 = (int)(hi4.x >> 16), sp2 = (int)(hi4.y & 0xFFFFu), sp3 = (int)(hi4.y >> 16), sp4 = (int)(hi4.z & 0xFFFFu);
    const int msg_o = (int)(hi4.w & 0xFFFFu), msg_l = (int)(hi4.w >> 16);
    r.host = Span{r.line + sp1 + 1, sp2 - sp1 - 1};
    r.app = Span{r.line + sp2 + 1, sp3 - sp2 - 1};
    r.proc = Span{r.line + sp3 + 1, sp4 - sp3 - 1};
    if (msg_l) r.msg = Span{r.line + msg_o, msg_l};
    r.full = Span{r.line, msg_o + msg_l};
    r.first = lo4.w;
    r.count = hi4.x & 0xFFFFu;
    if ((unsigned long long)r.first + r.count > (unsigned long long)P.entry_cap) { r.ok = false; return; }
    for (uint32_t e = r.first; e < r.first + r.count; ++e) {
        const unsigned long long v = P.entries[e];
        if (v & kE8Header) {
            r.has_sd = true;
            r.sd_id = Span{r.line + (int)(v & 0xFFFFu), (int)((v >> 16) & 0xFFFFu) - (int)(v & 0xFFFFu)};
        }
    }
}

constexpr uint32_t kMsgArena = 0x40u;    // FG_FLAG_MSG_ARENA: msg.x indexes the arena
constexpr uint32_t kNoSeverity = 0xFFu;  // a line without <PRI>: Record.severity is None

// An RFC3164 row: absolute spans (fg_parse3164.cu).  msg is never None: an empty message still gets a non-null pointer.
__device__ __forceinline__ void load_view_3164(const GelfEncodeParams& P, const ByteSource& B, int i, RecView& r) {
    const uint32_t meta = P.col_meta[i];
    r.ok = (meta & 0xFFu) == 0u;
    r.wide = false;
    r.has_sd = false;
    r.first = r.count = 0;
    if (!r.ok) return;
    r.severity = (meta >> 16) & 0xFFu;
    r.ts = P.col_ts[i];
    const int2 h = P.col_host[i], m = P.col_msg[i], f = P.col_full[i];
    r.host = Span{B.at(h.x), h.y};
    r.full = Span{B.at(f.x), f.y};
    if ((meta >> 24) & kMsgArena) {
        if ((unsigned long long)(uint32_t)m.x + (uint32_t)m.y > (unsigned long long)P.arena_cap) { r.ok = false; return; }
        r.msg = Span{P.arena + (uint32_t)m.x, m.y};
    } else {
        r.msg = Span{B.at(m.x), m.y};
    }
}

// An LTSV row: the column layout of RFC3164 (absolute spans, fg_parse_ltsv.cu) plus sd = its rows of the side table.
// msg.x < 0: the line has no `message` part (None, written "-"); `message:` is Some("") and gets a non-null pointer.
__device__ __forceinline__ void load_view_ltsv(const GelfEncodeParams& P, const ByteSource& B, int i, RecView& r) {
    const uint32_t meta = P.col_meta[i];
    r.ok = (meta & 0xFFu) == 0u;
    r.wide = false;
    r.has_sd = false;
    r.first = r.count = 0;
    if (!r.ok) return;
    r.severity = (meta >> 16) & 0xFFu;
    r.ts = P.col_ts[i];
    const int2 h = P.col_host[i], m = P.col_msg[i], f = P.col_full[i], sd = P.col_sd[i];
    r.host = Span{B.at(h.x), h.y};
    r.full = Span{B.at(f.x), f.y};
    r.msg = m.x >= 0 ? Span{B.at(m.x), m.y} : Span{nullptr, 0};
    r.first = (uint32_t)sd.x;
    r.count = (uint32_t)sd.y;
    if ((unsigned long long)r.first + r.count > (unsigned long long)P.wentry_cap) r.ok = false;
}

// pair e of the line (false: the row is an element header)
__device__ __forceinline__ bool load_pair(const GelfEncodeParams& P, const ByteSource& B, const RecView& r, uint32_t e, Span& name,
                                          Span& val) {
    if (r.wide) {
        const uint8_t m = P.wentry_meta[e];
        if ((m & 0x07u) == 7u) return false;
        name = Span{B.at(P.wentry_name[e].x), P.wentry_name[e].y};
        const unsigned long long v = P.wentry_val[e];
        val = Span{(m & 0x80u) ? P.arena + (uint32_t)v : B.at((int)(uint32_t)v), (int)(v >> 32)};
        return true;
    }
    const unsigned long long v = P.entries[e];
    if (v & kE8Header) return false;
    const int ns = (int)(v & 0xFFFFu), ne = (int)((v >> 16) & 0xFFFFu);
    name = Span{r.line + ns, ne - ns};
    if (v & kE8Arena) {
        const uint8_t* rec = P.arena + ((uint32_t)((v >> 32) & 0x3FFFFFFFu) << 1);
        val = Span{rec + 2, (int)*reinterpret_cast<const uint16_t*>(rec)};
    } else {
        val = Span{r.line + ne + 2, (int)((v >> 32) & 0xFFFFu) - (ne + 2)};
    }
    return true;
}

// An LTSV pair.  Its key after the '_' is name + suffix (ltsv_decoder.rs:131-193: the type's suffix when the entry has
// FG_EM_SUFFIX), so two different names can give the same key; tag 0: a string value (v = offset | length << 32), else
// the fg_ltsv_type of the 8 value bytes in v.
struct LtsvKey {
    Span name, suffix;
};
struct LtsvVal {
    unsigned long long v;
    uint32_t tag;
    uint32_t e;  // its row
};
constexpr uint32_t kEmSuffix = 0x20u;  // FG_EM_SUFFIX

__device__ __forceinline__ bool load_pair_ltsv(const GelfEncodeParams& P, const ByteSource& B, uint32_t e, LtsvKey& key, LtsvVal& val) {
    const uint32_t m = P.wentry_meta[e], t = m & 0x07u;
    const int2 nm = P.wentry_name[e];
    key.name = Span{B.at(nm.x), nm.y};
    key.suffix = Span{nullptr, 0};
    if (m & kEmSuffix) {
        const int a = P.ltsv_suffix_off[t];
        key.suffix = Span{P.ltsv_suffix + a, P.ltsv_suffix_off[t + 1] - a};
    }
    val.v = P.wentry_val[e];
    val.tag = t;
    val.e = e;
    return true;
}

// byte k of the composed key (after the '_')
__device__ __forceinline__ uint32_t key_byte(const LtsvKey& a, int k) {
    return k < a.name.len ? a.name.p[k] : a.suffix.p[k - a.name.len];
}
__device__ __forceinline__ int key_len(const LtsvKey& a) { return a.name.len + a.suffix.len; }
__device__ __forceinline__ uint32_t name_prefix(const LtsvKey& n) {
    uint32_t k = 0;
    for (int j = 0; j < 4; ++j) k = (k << 8) | (j < key_len(n) ? key_byte(n, j) : 0u);
    return k;
}
__device__ __forceinline__ int cmp_names(const LtsvKey& a, const LtsvKey& b) {
    const int la = key_len(a), lb = key_len(b), n = min(la, lb);
    for (int k = 0; k < n; ++k) {
        const uint32_t x = key_byte(a, k), y = key_byte(b, k);
        if (x != y) return x < y ? -1 : 1;
    }
    return la == lb ? 0 : (la < lb ? -1 : 1);
}
// byte-order comparison of ('_' + name + suffix) with b
__device__ __forceinline__ int cmp_sd_key(const LtsvKey& a, Span b) {
    if (b.len == 0) return 1;
    if ((uint32_t)'_' != b.p[0]) return (uint32_t)'_' < b.p[0] ? -1 : 1;
    const int la = key_len(a), n = min(la, b.len - 1);
    for (int k = 0; k < n; ++k) {
        const uint32_t x = key_byte(a, k), y = b.p[k + 1];
        if (x != y) return x < y ? -1 : 1;
    }
    return la == b.len - 1 ? 0 : (la < b.len - 1 ? -1 : 1);
}

// The record sources the kernels are instantiated for.  kSd: the record may carry structured data.  kOptional:
// application_name and process_id are None, and level is None without a severity.  kLtsv: pairs are LtsvKey / LtsvVal
// (composed keys, typed values), and the size pass writes the "Missing value" stop of every line.
struct From5424 {
    static constexpr bool kSd = true, kOptional = false, kLtsv = false;
    using Key = Span;
    using Val = Span;
    static __device__ __forceinline__ void load(const GelfEncodeParams& P, const ByteSource& B, int i, RecView& r) { load_view(P, B, i, r); }
    static __device__ __forceinline__ uint32_t status(const GelfEncodeParams& P, int i) { return P.rows[2 * (size_t)i].z & 0xFFu; }
    static __device__ __forceinline__ bool pair(const GelfEncodeParams& P, const ByteSource& B, const RecView& r, uint32_t e, Key& k, Val& v) {
        return load_pair(P, B, r, e, k, v);
    }
};
struct From3164 {
    static constexpr bool kSd = false, kOptional = true, kLtsv = false;
    using Key = Span;
    using Val = Span;
    static __device__ __forceinline__ void load(const GelfEncodeParams& P, const ByteSource& B, int i, RecView& r) { load_view_3164(P, B, i, r); }
    static __device__ __forceinline__ uint32_t status(const GelfEncodeParams& P, int i) { return P.col_meta[i] & 0xFFu; }
    static __device__ __forceinline__ bool pair(const GelfEncodeParams& P, const ByteSource& B, const RecView& r, uint32_t e, Key& k, Val& v) {
        return load_pair(P, B, r, e, k, v);
    }
};
struct FromLtsv {
    static constexpr bool kSd = true, kOptional = true, kLtsv = true;
    using Key = LtsvKey;
    using Val = LtsvVal;
    static __device__ __forceinline__ void load(const GelfEncodeParams& P, const ByteSource& B, int i, RecView& r) { load_view_ltsv(P, B, i, r); }
    static __device__ __forceinline__ uint32_t status(const GelfEncodeParams& P, int i) { return P.col_meta[i] & 0xFFu; }
    static __device__ __forceinline__ bool pair(const GelfEncodeParams& P, const ByteSource& B, const RecView&, uint32_t e, Key& k, Val& v) {
        return load_pair_ltsv(P, B, e, k, v);
    }
};

// ltsv_decoder.rs:99 prints "Missing value for name '{part}'" for every part without ':' the decode loop reached.  The
// stop of line i, relative to its start: -1 when nothing was printed, else the end of the parts that were read — the
// failing part's offset on an error row (fg_parse_ltsv.cu keeps it in full.x), the line's length + 1 otherwise.
constexpr uint32_t kMissingValue = 0x02u;  // FG_FLAG_MISSING_VALUE
__device__ __forceinline__ int32_t ltsv_stop(const GelfEncodeParams& P, int i) {
    const uint32_t meta = P.col_meta[i], st = meta & 0xFFu;
    if (!((meta >> 24) & kMissingValue) || st == FG_ES_INVALID_UTF8) return -1;  // a line that is not UTF-8 is not decoded
    const int2 f = P.col_full[i];
    return st ? f.x - P.offsets[i] : f.y + 1;
}

// static items (host-prepared, sorted by key, extras already override fixed keys of the same name)
enum { GF_APP = 0, GF_FULL, GF_HOST, GF_LEVEL, GF_PROC, GF_SDID, GF_SHORT, GF_TS, GF_VERSION, GF_EXTRA = 100 };

// ---- a record = a short list of segments, then ONE byte loop -------------------------------------------------------
// Emitting field by field with a byte loop per field made every lane of a warp sit in a different loop, a few of 32
// lanes active at a time.  Now a lane first lists its record as
// segments (pointer, length, copy / JSON-escape) — short, divergent — and then all 32 lanes run the SAME loop that
// produces one output byte per iteration from the current segment.
struct Seg {
    const uint8_t* p;
    int len;  // bit 31: JSON-escape the bytes
};
constexpr int kMaxSegs = 56;  // a record with more segments is emitted in several windows (rebuilt with `skip`)
constexpr int kEscBit = (int)0x80000000u;
__device__ const uint8_t kLit[] = "{}\",\"_\":\"\"unknown\"\"-\"\"1.1\"01234567";
//                                 0 1 2 3..5 6..8 9..17      18..20 21..25 26..33
enum { L_OPEN = 0, L_CLOSE = 1, L_QUOTE = 2, L_PAIR = 3 /* ,"_ */, L_MID = 6 /* ":" */, L_UNKNOWN = 9, L_DASH = 18, L_V11 = 21, L_DIGITS = 26 };

struct SegList {
    Seg s[kMaxSegs];
    int n = 0;     // segments held: those with running index in [skip, skip + kMaxSegs)
    int idx = 0;   // running index over the whole record
    int skip = 0;
    __device__ __forceinline__ void reset(int skip_) { n = 0; idx = 0; skip = skip_; }
    __device__ __forceinline__ void push(const uint8_t* p, int len, bool esc) {
        if (len <= 0) return;
        if (idx >= skip && n < kMaxSegs) {
            s[n].p = p;
            s[n].len = len | (esc ? kEscBit : 0);
            ++n;
        }
        ++idx;
    }
    __device__ __forceinline__ void lit(int at, int len) { push(kLit + at, len, false); }
    __device__ __forceinline__ void str(Span v) {
        lit(L_QUOTE, 1);
        push(v.p, v.len, true);
        lit(L_QUOTE, 1);
    }
    // a number whose text does not exist yet (LTSV): the segment points at its 8 value bytes in the side table and holds
    // its fg_ltsv_type as length; run_segments formats it when it reaches the segment
    __device__ __forceinline__ void num(const unsigned long long* at, uint32_t tag) { push((const uint8_t*)at, (int)tag, false); }
};

// `"_` is already out; the rest of an LTSV pair: `name suffix":` and its value (ltsv_decoder.rs:131-193: a typed value is
// an SDValue, written as serde_json writes Bool / F64 / I64 / U64)
__device__ __forceinline__ void ltsv_pair(const GelfEncodeParams& P, SegList& L, const ByteSource& B, const LtsvKey& k, const LtsvVal& v) {
    L.push(k.name.p, k.name.len, true);
    L.push(k.suffix.p, k.suffix.len, true);
    if (v.tag == 0u) {
        L.lit(L_MID, 3);  // ":"
        L.push(B.at((int)(uint32_t)v.v), (int)(v.v >> 32), true);
        L.lit(L_QUOTE, 1);
        return;
    }
    L.lit(L_MID, 2);  // ":
    L.num(P.wentry_val + v.e, v.tag);
}

// serde_json 0.8 for the typed values of an LTSV record: Bool as true / false, F64 through dtoa (non-finite -> null),
// I64 / U64 in decimal
__device__ __forceinline__ int json_number(unsigned long long v, uint32_t tag, uint8_t* out) {
    if (tag == 1u) {
        const uint32_t w = v ? 0x65757274u : 0x736C6166u;  // "true" / "fals", low byte first
        for (int k = 0; k < 4; ++k) out[k] = (uint8_t)(w >> (8 * k));
        out[4] = 'e';
        return v ? 4 : 5;
    }
    if (tag == 2u) return json_f64(__longlong_as_double((long long)v), out);
    int n = 0;
    if (tag == 3u && (long long)v < 0) {
        out[n++] = '-';
        v = 0ull - v;  // i64::MIN too
    }
    int d = 1;
    for (unsigned long long t = v; t >= 10ull; t /= 10ull) ++d;
    n += d;
    for (int k = n - 1; d > 0; --k, --d, v /= 10ull) out[k] = (uint8_t)('0' + (uint32_t)(v % 10ull));
    return n;
}

// SD pairs in BTreeMap order.  The pairs of a line are gathered once as (4-byte big-endian name prefix, row) and
// insertion-sorted by prefix (full byte compare only on equal prefixes; stable, so of equal names the LAST one — the one
// a later insert leaves in the map, gelf_encoder.rs:109 — closes its run).  Lines with more pairs than the local array
// holds fall back to selecting the next name by scanning all rows (O(pairs^2) full compares).
constexpr int kLocalPairs = 24;
struct PairRef {
    uint32_t key;
    uint32_t row;
};
__device__ __forceinline__ uint32_t name_prefix(Span n) {
    uint32_t k = 0;
    for (int j = 0; j < 4; ++j) k = (k << 8) | (j < n.len ? (uint32_t)n.p[j] : 0u);
    return k;
}

// (keys and values of the source's type: Span for RFC5424, LtsvKey / LtsvVal for LTSV)
template <class Src>
struct PairCursor {
    using Key = typename Src::Key;
    using Val = typename Src::Val;
    PairRef pr[kLocalPairs];
    int np = 0, at = 0;
    bool many = false;
    Key prev{nullptr, -1};
    bool have_prev = false;

    __device__ __forceinline__ void init(const GelfEncodeParams& P, const ByteSource& B, const RecView& r) {
        for (uint32_t e = r.first; e < r.first + r.count; ++e) {
            Key nm;
            Val vl;
            if (!Src::pair(P, B, r, e, nm, vl)) continue;
            if (np == kLocalPairs) { many = true; break; }
            const uint32_t key = name_prefix(nm);
            int j = np++;
            while (j > 0) {  // stable insertion: move entries that sort strictly after the new one
                const PairRef q = pr[j - 1];
                bool after = q.key > key;
                if (q.key == key) {
                    Key qn;
                    Val qv;
                    Src::pair(P, B, r, q.row, qn, qv);
                    after = cmp_names(qn, nm) > 0;
                }
                if (!after) break;
                pr[j] = q;
                --j;
            }
            pr[j].key = key;
            pr[j].row = e;
        }
    }
    // next pair in key order with duplicates resolved; false when exhausted
    __device__ __forceinline__ bool next(const GelfEncodeParams& P, const ByteSource& B, const RecView& r, Key& bn, Val& bv) {
        if (!many) {
            while (at < np) {
                Src::pair(P, B, r, pr[at].row, bn, bv);
                ++at;
                if (at < np && pr[at].key == pr[at - 1].key) {  // a later pair with the same name replaces this one
                    Key nn;
                    Val nv;
                    Src::pair(P, B, r, pr[at].row, nn, nv);
                    if (cmp_names(nn, bn) == 0) continue;
                }
                return true;
            }
            return false;
        }
        bool have = false;
        for (uint32_t e = r.first; e < r.first + r.count; ++e) {
            Key nm;
            Val vl;
            if (!Src::pair(P, B, r, e, nm, vl)) continue;
            if (have_prev && cmp_names(nm, prev) <= 0) continue;
            if (!have || cmp_names(nm, bn) <= 0) {
                bn = nm;
                bv = vl;
                have = true;
            }
        }
        return have;
    }
    __device__ __forceinline__ void taken(Key bn) {
        prev = bn;
        have_prev = true;
    }
};

// `num` (>= 32 bytes, owned by the caller) receives the text of Record.ts and is referenced by a segment.
// Called by ALL 32 lanes (`live` = this lane has a record).  The loop runs over the STATIC items, which are the same for
// every record, so the lanes of a warp stay on the same item (the first version merged pair by pair per lane: the lanes
// drifted apart by their pair counts and every static item ran a few lanes wide); the SD pairs that
// sort before the current item are emitted by an inner loop whose trip count is the warp's maximum.
template <class Src>
__device__ __forceinline__ void build_segments(const GelfEncodeParams& P, const ByteSource& B, const RecView& r, bool live, uint8_t* num,
                                               SegList& L) {
    if (live) L.lit(L_OPEN, 1);
    bool first = true;
    PairCursor<Src> pc;
    if (Src::kSd && live) pc.init(P, B, r);
    typename Src::Key bn{nullptr, 0};
    typename Src::Val bv{};
    bool have = Src::kSd && live && pc.next(P, B, r, bn, bv);
    for (int si = 0; si <= P.n_static; ++si) {  // warp-uniform; si == n_static: the pairs after the last static item
        const bool tail = si == P.n_static;
        Span key{nullptr, 0};
        if (!tail) key = Span{P.static_blob + P.static_key_off[si], P.static_key_off[si + 1] - P.static_key_off[si]};
        int c = 1;
        for (;;) {
            c = have ? (tail ? -1 : cmp_sd_key(bn, key)) : 1;
            const bool emit = have && c < 0;
            if (!__any_sync(0xFFFFFFFFu, emit)) break;
            if (emit) {
                L.lit(L_PAIR + (first ? 1 : 0), first ? 2 : 3);  // ,"_
                first = false;
                if constexpr (Src::kLtsv) {
                    ltsv_pair(P, L, B, bn, bv);
                } else {
                    L.push(bn.p, bn.len, true);
                    L.lit(L_MID, 3);  // ":"
                    L.push(bv.p, bv.len, true);
                    L.lit(L_QUOTE, 1);
                }
                pc.taken(bn);
                have = pc.next(P, B, r, bn, bv);
            }
        }
        if (tail) break;
        const int kind = P.static_kind[si];
        if (live) {
            bool take = true;
            if (c == 0) {
                if (kind == GF_EXTRA) {  // extras are inserted last (gelf_encoder.rs:110-112): the SD pair of this key is dropped
                    pc.taken(bn);
                    have = pc.next(P, B, r, bn, bv);
                } else {
                    take = false;  // an SD pair replaces a fixed field of the same key: the next round's pair loop emits it
                }
            }
            if (kind == GF_SDID && !r.has_sd) take = false;
            if (Src::kOptional && (kind == GF_APP || kind == GF_PROC || (kind == GF_LEVEL && r.severity == kNoSeverity))) take = false;
            if (take) {
                // the literal is `,"key":` (for an extra `,"key":"value"`): the comma is skipped for the first item
                const uint8_t* lit = P.static_blob + P.static_lit_off[si];
                const int lit_len = P.static_lit_off[si + 1] - P.static_lit_off[si];
                L.push(lit + (first ? 1 : 0), lit_len - (first ? 1 : 0), false);
                first = false;
                switch (kind) {  // warp-uniform
                    case GF_APP: L.str(r.app); break;
                    case GF_FULL: L.str(r.full); break;
                    case GF_HOST:
                        if (r.host.len == 0) L.lit(L_UNKNOWN, 9);
                        else L.str(r.host);
                        break;
                    case GF_LEVEL: L.lit(L_DIGITS + (int)(r.severity & 7u), 1); break;
                    case GF_PROC: L.str(r.proc); break;
                    case GF_SDID: L.str(r.sd_id); break;
                    case GF_SHORT:
                        if (r.msg.p == nullptr) L.lit(L_DASH, 3);
                        else L.str(r.msg);
                        break;
                    case GF_TS: L.push(num, json_f64(r.ts, num), false); break;
                    case GF_VERSION: L.lit(L_V11, 5); break;
                    default: break;  // GF_EXTRA: the literal was everything
                }
            }
        }
    }
    if (live) L.lit(L_CLOSE, 1);
}

// serde_json 0.8 ser.rs escape_bytes: `"` `\` \b \f \n \r \t get a backslash form (returns the second byte), else 0
__device__ __forceinline__ uint32_t json_escape_of(uint32_t c) {
    if (c == '"' || c == '\\') return c;
    if (c >= 0x20u) return 0u;
    return c == 8u ? 'b' : c == 9u ? 't' : c == 10u ? 'n' : c == 12u ? 'f' : c == 13u ? 'r' : 0u;
}

// 0x80 in every byte of w that serde_json escapes: '"', '\\', or a byte below 0x20 (a superset of \b \f \n \r \t: the
// other control bytes take the one-byte path and are copied there)
__device__ __forceinline__ uint32_t json_escape_flags4(uint32_t w) {
    const uint32_t x1 = w ^ 0x22222222u, x2 = w ^ 0x5C5C5C5Cu, t = w & 0xE0E0E0E0u;
    const uint32_t n1 = ((x1 & 0x7F7F7F7Fu) + 0x7F7F7F7Fu) | x1, n2 = ((x2 & 0x7F7F7F7Fu) + 0x7F7F7F7Fu) | x2,
                   n3 = ((t & 0x7F7F7F7Fu) + 0x7F7F7F7Fu) | t;  // bit 7: byte != 0
    return ~(n1 & n2 & n3) & 0x80808080u;
}

// The warp-uniform loop: per lane and iteration FOUR output bytes when the segment has them and none needs an escape, else
// one.  `live` = this lane has a record to emit.  (One byte per iteration spends the loop's bookkeeping on every byte.)
// kNum (Sink = NumSink): the list may hold number segments, formatted into `text` when the loop enters them (segments are
// consumed in order, so one buffer serves all the numbers of a record).
template <class Sink, bool kNum = false>
__device__ __forceinline__ void run_segments(const SegList& L, bool live, Sink& s) {
    int si = 0, k = 0, len = 0;
    bool esc = false;
    const uint8_t* p = nullptr;
    uint32_t pending = 0;
    bool more = live && L.n > 0;
    uint8_t text[kNum ? 32 : 1];
    auto enter_number = [&]() {
        if constexpr (kNum) {
            const unsigned long long* v = reinterpret_cast<const unsigned long long*>(p);
            if (v >= s.vals && v < s.vals + s.cap) {  // no byte segment points into the value column
                len = json_number(*v, (uint32_t)len, text);
                p = text;
            }
        }
    };
    if (more) {
        p = L.s[0].p;
        len = L.s[0].len & ~kEscBit;
        esc = L.s[0].len < 0;
        enter_number();
    }
    while (__any_sync(0xFFFFFFFFu, more)) {
        if (more) {
            uint32_t w;
            int n = 1;
            if (pending) {
                w = pending;
                pending = 0;
            } else {
                w = p[k];
                if (k + 4 <= len) {
                    const uint32_t w4 = w | ((uint32_t)p[k + 1] << 8) | ((uint32_t)p[k + 2] << 16) | ((uint32_t)p[k + 3] << 24);
                    if (!esc || json_escape_flags4(w4) == 0u) {
                        w = w4;
                        n = 4;
                    }
                }
                k += n;
                if (esc && n == 1) {
                    const uint32_t e = json_escape_of(w);
                    if (e) { pending = e; w = '\\'; }
                }
            }
            s.push(w, n);
            if (k >= len && !pending) {  // next segment (none is empty)
                ++si;
                if (si < L.n) {
                    p = L.s[si].p;
                    len = L.s[si].len & ~kEscBit;
                    esc = L.s[si].len < 0;
                    k = 0;
                    enter_number();
                } else {
                    more = false;
                }
            }
        }
    }
}

// a record of any size: windows of kMaxSegs segments, every window through the warp-uniform loop
template <class Src, class Sink>
__device__ __forceinline__ void emit_record(const GelfEncodeParams& P, const ByteSource& B, const RecView& r, bool live, Sink& s) {
    uint8_t num[32];
    SegList L;
    int skip = 0;
    for (;;) {
        L.reset(skip);
        build_segments<Src>(P, B, r, live, num, L);
        if constexpr (Src::kLtsv) {
            NumSink<Sink> ns{s, P.wentry_val, P.wentry_cap};
            run_segments<NumSink<Sink>, true>(L, live, ns);
        } else {
            run_segments(L, live, s);
        }
        skip += kMaxSegs;
        if (!__any_sync(0xFFFFFFFFu, live && L.idx > skip)) break;
    }
    if (live) s.finish();
}

// Both kernels stage the byte span of the CTA's lines in shared memory with one TMA bulk copy, like the parse kernel:
// a lane reading ITS line byte by byte from global memory would cost 32 L1 wavefronts per load instruction (32 lanes,
// 32 different lines); from the tile it is one shared-memory access.  A span larger than the tile is read from global.
//
// The byte loop of a warp runs as long as its LONGEST record, and record lengths follow the line lengths (full_message
// is the line, short_message its tail): with lines in input order a warp ran ~4x longer than its mean record.  So a CTA
// takes 256 lines and hands them to its threads in order of line length (counting sort over 16-byte classes): the 32
// lines of a warp are neighbours in length.  Which thread emits which line changes nothing in the output.
constexpr int kEncLines = 256;
constexpr int kLenClasses = 64;

struct EncShared {
    uint64_t mbar;
    uint32_t hist[kLenClasses];
    uint16_t perm[kEncLines];
};

__device__ __forceinline__ ByteSource stage_lines(const GelfEncodeParams& P, uint8_t* tile, uint64_t* mbar, int first, int last) {
    TileStage stage = {mbar};
    stage.init();
    const int base = span_base(P.offsets[first]);
    const uint32_t nbytes = span_copy_bytes(base, P.offsets[last]);
    if (nbytes <= (uint32_t)P.tile_bytes) {  // CTA-uniform
        __syncthreads();                     // the barrier is initialised before anyone arrives or waits on it
        stage.load(tile, P.bytes + base, nbytes);
        return ByteSource{tile, base};
    }
    return ByteSource{P.bytes, 0};
}

// line handled by this thread: the CTA's lines in order of length class (-1: none)
__device__ __forceinline__ int sorted_line(const GelfEncodeParams& P, EncShared& sh, int first, int last) {
    const int tid = threadIdx.x;
    if (tid < kLenClasses) sh.hist[tid] = 0;
    __syncthreads();
    const int i = first + tid;
    uint32_t cls = 0, rank = 0;
    if (i < last) {
        cls = min((uint32_t)(P.offsets[i + 1] - P.offsets[i]) >> 4, (uint32_t)kLenClasses - 1u);
        rank = atomicAdd(&sh.hist[cls], 1u);
    }
    __syncthreads();
    if (tid < 32) {  // exclusive scan of the 64 class counts by one warp (two classes per lane)
        const uint32_t a = sh.hist[2 * tid], b = sh.hist[2 * tid + 1];
        uint32_t x = a + b;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
            const uint32_t y = __shfl_up_sync(0xFFFFFFFFu, x, d);
            if (tid >= d) x += y;
        }
        sh.hist[2 * tid] = x - a - b;
        sh.hist[2 * tid + 1] = x - b;
    }
    __syncthreads();
    if (i < last) sh.perm[sh.hist[cls] + rank] = (uint16_t)tid;
    __syncthreads();
    return tid < last - first ? first + (int)sh.perm[tid] : -1;
}

template <class Src>
__global__ void __launch_bounds__(kEncLines) gelf_size_kernel(const __grid_constant__ GelfEncodeParams P) {
    extern __shared__ __align__(128) uint8_t tile[];
    __shared__ __align__(8) EncShared sh;
    if (*P.bad_offsets) return;
    const int first = blockIdx.x * kEncLines, last = min(P.n, first + kEncLines);
    const ByteSource B = stage_lines(P, tile, &sh.mbar, first, last);
    const int i = sorted_line(P, sh, first, last);
    const bool valid = i >= 0;
    RecView r;
    r.ok = false;
    if (valid) Src::load(P, B, i, r);
    CountSink s;
    emit_record<Src>(P, B, r, r.ok, s);
    if (!valid) return;
    P.lens[i] = r.ok ? s.n : 0ull;
    P.status[i] = (uint8_t)Src::status(P, i);
    if constexpr (Src::kLtsv) P.ltsv_stop[i] = ltsv_stop(P, i);
}

// chunk totals: base[k + 1] = base[k] + bytes of this chunk (one thread)
__global__ void gelf_base_kernel(const __grid_constant__ GelfEncodeParams P) {
    if (*P.bad_offsets) return;
    const unsigned long long total = P.rel[P.n - 1] + P.lens[P.n - 1];
    P.base[1] = P.base[0] + total;
}

template <class Src>
__global__ void __launch_bounds__(kEncLines) gelf_write_kernel(const __grid_constant__ GelfEncodeParams P) {
    extern __shared__ __align__(128) uint8_t tile[];
    __shared__ __align__(8) EncShared sh;
    if (*P.bad_offsets) return;
    const int first = blockIdx.x * kEncLines, last = min(P.n, first + kEncLines);
    const ByteSource B = stage_lines(P, tile, &sh.mbar, first, last);
    const int i = sorted_line(P, sh, first, last);
    const bool valid = i >= 0;
    unsigned long long at = 0, len = 0;
    if (valid) {
        at = P.base[0] + P.rel[i];
        len = P.lens[i];
        P.out_offsets[i] = (long long)at;
        if (i == P.n - 1) P.out_offsets[P.n] = (long long)(at + len);
    }
    // a rejected line has no record; an output buffer that overflowed is not written (the batch is redone)
    const bool live = valid && len != 0ull && at + len <= P.out_cap;
    RecView r;
    r.ok = false;
    if (live) Src::load(P, B, i, r);
    WordSink s(P.out + at);
    emit_record<Src>(P, B, r, live && r.ok, s);
}

template <class Src>
cudaError_t configure_src(int max_tile_bytes) {
    cudaError_t e = cudaFuncSetAttribute(gelf_size_kernel<Src>, cudaFuncAttributeMaxDynamicSharedMemorySize, max_tile_bytes);
    if (e != cudaSuccess) return e;
    return cudaFuncSetAttribute(gelf_write_kernel<Src>, cudaFuncAttributeMaxDynamicSharedMemorySize, max_tile_bytes);
}

template <class Src>
cudaError_t launch_src(const GelfEncodeParams& p, void* d_scan_temp, size_t scan_temp_bytes, cudaStream_t stream) {
    const int grid = (p.n + kEncLines - 1) / kEncLines;
    gelf_size_kernel<Src><<<grid, kEncLines, p.tile_bytes, stream>>>(p);
    cudaError_t e = cub::DeviceScan::ExclusiveSum(d_scan_temp, scan_temp_bytes, p.lens, p.rel, p.n, stream);
    if (e != cudaSuccess) return e;
    gelf_base_kernel<<<1, 1, 0, stream>>>(p);
    gelf_write_kernel<Src><<<grid, kEncLines, p.tile_bytes, stream>>>(p);
    return cudaGetLastError();
}

}  // namespace

// every source gets the same staging limit: launch_encode clamps every tile to it
cudaError_t configure_gelf_encode(int max_tile_bytes) {
    cudaError_t e = configure_src<From5424>(max_tile_bytes);
    if (e != cudaSuccess) return e;
    e = configure_src<From3164>(max_tile_bytes);
    if (e != cudaSuccess) return e;
    return configure_src<FromLtsv>(max_tile_bytes);
}

size_t gelf_scan_temp_bytes(int n) {
    size_t bytes = 0;
    cub::DeviceScan::ExclusiveSum(nullptr, bytes, (const unsigned long long*)nullptr, (unsigned long long*)nullptr, n);
    return bytes;
}

cudaError_t launch_gelf_encode(int fmt, const GelfEncodeParams& p, void* d_scan_temp, size_t scan_temp_bytes, cudaStream_t stream) {
    if (p.n <= 0) return cudaSuccess;
    switch (fmt) {
        case 0: return launch_src<From5424>(p, d_scan_temp, scan_temp_bytes, stream);
        case 1: return launch_src<FromLtsv>(p, d_scan_temp, scan_temp_bytes, stream);
        case 3: return launch_src<From3164>(p, d_scan_temp, scan_temp_bytes, stream);
        default: return cudaErrorInvalidValue;
    }
}

}  // namespace fg
