// fg_gelf_encode.cu — the stage AFTER the decoder, fused on the device: Record -> GELF JSON bytes (SURVEY.md §8(f) N2).
//
// H100-native replacement for GelfEncoder::encode (flowgger src/flowgger/encoder/gelf_encoder.rs:59-115), which
// every splitter calls right after Decoder::decode (splitter/line_splitter.rs:50-52).  The JSON text is what
// serde_json "~0.8" `to_vec` prints for the BTreeMap the reference builds: keys in byte order, a later insert replaces
// an earlier one (SD pairs replace fixed fields, output.gelf_extra replaces everything), compact separators, strings
// with `"` `\\` \b \f \n \r \t escaped, Record.ts through dtoa (fg_dtoa.cuh).
//
// Input = the decoder's device-resident results; nothing of them travels to the host in this mode.  Four record
// sources, chosen at compile time (the kernels are templates on the source, everything after the record view is shared):
//   From5424  compact rows + 8-byte entries + arena, or wide rows (structured data; every fixed field present)
//   From3164  the row columns of parse3164_kernel + the arena of re-joined messages (rfc3164_decoder.rs:71-82, 106-117:
//             no appname, procid or structured data; no severity without <PRI>; msg always Some, possibly "")
//   FromLtsv  the row columns of parse_ltsv_kernel + its 17-byte side table (ltsv_decoder.rs:87-221: no appname, procid
//             or sd_id; no severity without `level`; msg None without `message`).  A pair's key is '_' + name + the
//             type's suffix (FG_EM_SUFFIX), so keys are ordered and de-duplicated on that composed text; a typed value
//             (bool, f64, i64, u64) is written as JSON, not as its source text.
//   FromGelf  the row columns of parse_gelf_kernel / post_gelf_kernel + their 17-byte side table (gelf_decoder.rs:34-125:
//             no appname, procid or sd_id; level, short_message and full_message only when the object has them; the
//             wall clock of the call for a record without "timestamp").  A member's key is '_' + its name (the name alone
//             when it starts with '_', FG_EM_NO_PREFIX); names, strings and keys are compared and written as their
//             UNESCAPED text: a span that holds JSON escapes is re-encoded through the decoder's own KeyIter.
// Launches per chunk of lines:
//   gelf_size_kernel   one thread per line: exact length of its record (0 for a line the decoder rejected); the bytes of
//                      the CTA's 256 lines are staged in shared memory by one TMA bulk copy and handed to the threads
//                      in order of line length (both kernels)
//   cub exclusive sum  record offsets inside the chunk
//   gelf_write_kernel  one thread per line writes its record; output bytes are assembled four at a time and stored as
//                      aligned 32-bit words, so a record costs a quarter of the store instructions / L2 requests of a
//                      byte-wise copy
// Both kernels run ONE emit routine over a counting or a writing sink, so the two passes cannot disagree.  output.framing
// (fg_out_frame.cuh) is one runtime value: the size pass counts the frame into a record's length, the write pass stores
// the frame around the record's place before the record is emitted into it.
// All SD names start with '_' (rfc5424_decoder.rs:221), i.e. they sort before every fixed GELF key; the general merge
// with the pre-sorted static items (fixed keys + extras, prepared on the host once) still compares full keys.
#include <cub/device/device_scan.cuh>

#include "fg_dtoa.cuh"
#include "fg_encode_view.cuh"
#include "fg_out_frame.cuh"

namespace fg {

namespace {

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

// the unescaped bytes of a key, -1 at the end
struct KeyText {
    KeyIter it;
    __device__ __forceinline__ explicit KeyText(const GelfKey& a) { key_iter_init(it, a.name.p, 0, a.name.len, a.mode2); }
    __device__ __forceinline__ int next() { return key_iter_next(it); }
};
__device__ __forceinline__ uint32_t name_prefix(const GelfKey& n) {
    uint32_t k = 0;
    if (!n.esc) {
        for (int j = 0; j < 4; ++j) k = (k << 8) | (j < n.name.len ? (uint32_t)n.name.p[j] : 0u);
        return k;
    }
    KeyText t(n);
    for (int j = 0; j < 4; ++j) {
        const int c = t.next();
        k = (k << 8) | (c < 0 ? 0u : (uint32_t)c);
        if (c < 0) {
            k <<= 8 * (3 - j);
            break;
        }
    }
    return k;
}
__device__ __forceinline__ int cmp_names(const GelfKey& a, const GelfKey& b) {
    if (!a.esc && !b.esc) return cmp_names(a.name, b.name);
    KeyText x(a), y(b);
    for (;;) {
        const int cx = x.next(), cy = y.next();
        if (cx != cy) return cx < cy ? -1 : 1;
        if (cx < 0) return 0;
    }
}
// byte-order comparison of ('_' + key) with b
__device__ __forceinline__ int cmp_sd_key(const GelfKey& a, Span b) {
    if (!a.esc) return cmp_sd_key(a.name, b);
    if (b.len == 0) return 1;
    if ((uint32_t)'_' != b.p[0]) return (uint32_t)'_' < b.p[0] ? -1 : 1;
    KeyText x(a);
    for (int k = 1;; ++k) {
        const int cx = x.next(), cy = k < b.len ? (int)b.p[k] : -1;
        if (cx != cy) return cx < cy ? -1 : 1;
        if (cx < 0) return 0;
    }
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
    int len;  // bit 31: JSON-escape the bytes; bit 30 (GELF): the bytes are a JSON string body, re-encoded step by step
};
constexpr int kMaxSegs = 56;  // a record with more segments is emitted in several windows (rebuilt with `skip`)
constexpr int kEscBit = (int)0x80000000u;
constexpr int kJsonBit = 0x40000000;
constexpr int kMaxSegLen = kJsonBit - 1;  // the longest span one segment holds
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
    // GELF: a string span as serde_json writes its unescaped text; json = the span holds JSON escapes.  A span longer than
    // kMaxSegLen is cut into several segments, which is exact because the escapes of a copied span are per byte (the
    // other sources need no cut: their byte loop reads bit 30 as length).  A span with JSON escapes is not cut (a cut
    // could split an escape): long_json_span_kernel fails the call for one that long.
    __device__ __forceinline__ void text(const uint8_t* p, int len, bool json) {
        if (!json) {
            for (; len > kMaxSegLen; p += kMaxSegLen, len -= kMaxSegLen) push(p, kMaxSegLen, true);
            push(p, len, true);
        } else if (len > 0) {
            push(p, len | kJsonBit, true);
        }
    }
    __device__ __forceinline__ void str_json(Span v, bool json) {
        lit(L_QUOTE, 1);
        text(v.p, v.len, json);
        lit(L_QUOTE, 1);
    }
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

// `"_` is already out; the rest of a GELF member: `key":` and its value (gelf_decoder.rs:91-104: the JSON value as
// an SDValue, a string as its unescaped text)
__device__ __forceinline__ void gelf_pair(const GelfEncodeParams& P, SegList& L, const ByteSource& B, const GelfKey& k, const GelfVal& v) {
    L.text(k.name.p, k.name.len, k.esc);
    if (v.tag == 0u) {
        L.lit(L_MID, 3);  // ":"
        L.text(B.at((int)(uint32_t)v.v), (int)(v.v >> 32), v.esc);
        L.lit(L_QUOTE, 1);
        return;
    }
    L.lit(L_MID, 2);  // ":
    L.num(P.wentry_val + v.e, v.tag);
}

// serde_json 0.8 for the typed values of an LTSV or GELF record: Bool as true / false, F64 through dtoa (non-finite ->
// null), I64 / U64 in decimal; kNull (GELF): FG_TAG_NULL as null
template <bool kNull = false>
__device__ __forceinline__ int json_number(unsigned long long v, uint32_t tag, uint8_t* out) {
    if (kNull && tag == 5u) {
        const uint32_t w = 0x6C6C756Eu;  // "null", low byte first
        for (int k = 0; k < 4; ++k) out[k] = (uint8_t)(w >> (8 * k));
        return 4;
    }
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
                } else if constexpr (Src::kGelf) {
                    gelf_pair(P, L, B, bn, bv);
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
        int kind = P.static_kind[si];
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
            if constexpr (Src::kGelf) {
                if (kind == GF_FULL && r.full.p == nullptr) take = false;
            }
            if (take) {
                // the literal is `,"key":` (for an extra `,"key":"value"`): the comma is skipped for the first item
                const uint8_t* lit = P.static_blob + P.static_lit_off[si];
                const int lit_len = P.static_lit_off[si + 1] - P.static_lit_off[si];
                L.push(lit + (first ? 1 : 0), lit_len - (first ? 1 : 0), false);
                first = false;
                if constexpr (Src::kGelf) {  // the fixed string fields may hold JSON escapes
                    switch (kind) {
                        case GF_FULL: L.str_json(r.full, r.flags & kFullEsc); kind = -1; break;
                        case GF_HOST:
                            if (r.host.len) { L.str_json(r.host, r.flags & kHostEsc); kind = -1; }
                            break;
                        case GF_SHORT:
                            if (r.msg.p) { L.str_json(r.msg, r.flags & kMsgEsc); kind = -1; }
                            break;
                        default: break;
                    }
                }
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

// (json_escape_of, serde_json 0.8 ser.rs escape_bytes, lives in fg_gelf.cuh next to the decoder's unescape)

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

// The same loop for a GELF record, whose list may also hold JSON string bodies (kJsonBit; `mode2` = the line went
// through the newline retry): four source bytes per iteration while they hold no backslash and no byte to escape, else
// one source escape (or byte) re-encoded by json_transcode_step, 1..4 output bytes.  Numbers as in run_segments<kNum>,
// plus FG_TAG_NULL.  (A separate routine: any change to run_segments' template moves the register allocation of the
// other three sources' kernels.)
template <class Sink>
__device__ __forceinline__ void run_json_segments(const SegList& L, bool live, Sink& s, bool mode2) {
    int si = 0, k = 0, len = 0;
    bool esc = false, json = false;
    const uint8_t* p = nullptr;
    uint32_t pending = 0;
    bool more = live && L.n > 0;
    uint8_t text[32];
    auto enter = [&](const Seg& g) {
        p = g.p;
        len = g.len & ~(kEscBit | kJsonBit);
        esc = g.len < 0;
        json = (g.len & kJsonBit) != 0;
        k = 0;
        const unsigned long long* v = reinterpret_cast<const unsigned long long*>(p);
        if (v >= s.vals && v < s.vals + s.cap) {  // no byte segment points into the value column
            len = json_number<true>(*v, (uint32_t)len, text);
            p = text;
        }
    };
    if (more) enter(L.s[0]);
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
                if (json && n == 1) {
                    n = json_transcode_step(p, k, len, mode2, w);
                } else {
                    k += n;
                    if (esc && n == 1) {
                        const uint32_t e = json_escape_of(w);
                        if (e) { pending = e; w = '\\'; }
                    }
                }
            }
            s.push(w, n);
            if (k >= len && !pending) {  // next segment (none is empty)
                if (++si < L.n) enter(L.s[si]);
                else more = false;
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
        } else if constexpr (Src::kGelf) {
            NumSink<Sink> ns{s, P.wentry_val, P.wentry_cap};
            run_json_segments(L, live, ns, (r.flags & kNlRetry) != 0u);
        } else {
            run_segments(L, live, s);
        }
        skip += kMaxSegs;
        if (!__any_sync(0xFFFFFFFFu, live && L.idx > skip)) break;
    }
    if (live) s.finish();
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
    P.lens[i] = r.ok ? framed_len(s.n, P.out_framing) : 0ull;
    P.status[i] = (uint8_t)Src::status(P, i);
    if constexpr (Src::kLtsv) P.ltsv_stop[i] = ltsv_stop(P, i);
}
template <class Src>
__global__ void __launch_bounds__(kEncLines, Src::kWriteCtas) gelf_write_kernel(const __grid_constant__ GelfEncodeParams P) {
    extern __shared__ __align__(128) uint8_t tile[];
    __shared__ __align__(8) EncShared sh;
    if (*P.bad_offsets) return;
    const int first = blockIdx.x * kEncLines, last = min(P.n, first + kEncLines);
    if (P.out_framing != kOutNone && first + (int)threadIdx.x < last) {
        // output.framing of line first + tid, stored before any record of the CTA is emitted (a record's own bytes lie
        // strictly between its prefix and its suffix) and before the lines are sorted: none of it is live in the byte loop
        const int j = first + (int)threadIdx.x;
        const unsigned long long fl = P.lens[j], a = P.base[0] + P.rel[j];
        uint32_t pre = 0;
        if (fl != 0ull && a + fl <= P.out_cap) pre = (uint32_t)(frame_record(P.out_framing, fl, P.out + a) - (P.out + a));
        sh.pre[threadIdx.x] = (uint8_t)pre;
    }
    const ByteSource B = stage_lines(P, tile, &sh.mbar, first, last);
    const int i = sorted_line(P, sh, first, last);  // (its barriers publish sh.pre)
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
    WordSink s(P.out + at + (live && P.out_framing == kOutSyslen ? sh.pre[i - first] : 0));
    emit_record<Src>(P, B, r, live && r.ok, s);
}

template <class Src>
cudaError_t configure_src(int max_tile_bytes) {
    return configure_passes(gelf_size_kernel<Src>, gelf_write_kernel<Src>, max_tile_bytes);
}

template <class Src>
cudaError_t launch_src(const GelfEncodeParams& p, void* d_scan_temp, size_t scan_temp_bytes, cudaStream_t stream) {
    return launch_passes(gelf_size_kernel<Src>, gelf_write_kernel<Src>, p, d_scan_temp, scan_temp_bytes, stream);
}

}  // namespace

// every source gets the same staging limit: launch_encode clamps every tile to it
cudaError_t configure_gelf_encode(int max_tile_bytes) {
    cudaError_t e = configure_src<From5424>(max_tile_bytes);
    if (e != cudaSuccess) return e;
    e = configure_src<From3164>(max_tile_bytes);
    if (e != cudaSuccess) return e;
    e = configure_src<FromLtsv>(max_tile_bytes);
    if (e != cudaSuccess) return e;
    return configure_src<FromGelf>(max_tile_bytes);
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
        case 2:
            if (p.long_json_span) long_json_span_kernel<<<(p.n + kEncLines - 1) / kEncLines, kEncLines, 0, stream>>>(p, kMaxSegLen);
            return launch_src<FromGelf>(p, d_scan_temp, scan_temp_bytes, stream);
        case 3: return launch_src<From3164>(p, d_scan_temp, scan_temp_bytes, stream);
        default: return cudaErrorInvalidValue;
    }
}

}  // namespace fg
