// fg_capnp_encode.cu — the Cap'n Proto encoder fused after the decoder on the device: Record -> one serialized message
// (output.format = "capnp").
//
// H100-native replacement for CapnpEncoder::encode (flowgger src/flowgger/encoder/capnp_encoder.rs:36-109, record.capnp).
// A Record is a struct of 2 data words (ts as f64; facility, severity as u8 at bytes 8 and 9, 0xFF: None) and 9 pointers
// (hostname, appname, procid, msgid, msg, fullMsg, sdId, pairs, extra).  The objects are allocated in build_record's
// order: hostname; appname, procid, msgid, msg, full_msg when Some; of the FIRST SD element its id when Some and its
// pairs (a list of Pair structs, then each pair's key and string value); output.capnp_extra as a second pair list.
// A Pair is 2 data words (union discriminant string 0 / bool 1 / f64 2 / i64 3 / u64 4 / null 5 at byte 0, the bool
// at bit 16, the number in word 1) and 2 pointers (key, string value).  Pair keys are the Record's names: '_' + name
// (+ the LTSV type suffix); extras' keys are used as given.  Nothing is formatted or escaped: a text is its bytes, a
// NUL and zero bytes to the next word; a GELF string with JSON escapes is written unescaped.
//
// fg_capnp_layout.cuh places each object (the first segment, or landing pads and new segments past its 1024 words).  A
// record becomes a list of segments in output order — the segment table, then each message segment's words in
// allocation order — and all lanes of a warp run one byte loop over their lists, as the LTSV encoder does: computed
// words (pointers, data, tags, the table) 8 bytes in two pushes, text four bytes per iteration, a GELF span with
// escapes one unescape step at a time, and the NUL and zero pad to the next word.  Only the size pass knows no list:
// it places the objects and sums the words.  The record view, the sinks, the staging and the launch sequence are the
// other encoders' (fg_encode_view.cuh).
#include "fg_capnp_layout.cuh"
#include "fg_encode_view.cuh"
#include "fg_out_frame.cuh"

namespace fg {

namespace {

// the kind of a segment, read from its 32-bit length word: 0 is a NUL and pad (CK_END), all ones a computed word
// (CK_WORD), bit 31 a GELF span with JSON escapes (CK_JSON), else raw bytes.  A span holds less than 2^31 bytes, so a
// length holds any span a line can hold, also the raw JSON of a GELF string whose unescaped text capnp holds.
enum : uint32_t { CK_WORD = 0, CK_RAW = 1, CK_JSON = 2, CK_END = 3 };
constexpr uint32_t kLenEnd = 0u, kLenWord = 0xFFFFFFFFu, kLenJson = 1u << 31;

__device__ const uint8_t kUnderscore[] = "_";

// Record's pointer slots; a field text's slot is its index in CapRec::f
enum { CP_HOST = 0, CP_APP, CP_PROC, CP_MSGID, CP_MSG, CP_FULL, CP_SDID, CP_PAIRS, CP_EXTRA, CP_COUNT };

constexpr int kMaxCapSegs = 64;  // a record with more segments is emitted in several windows (rebuilt with `skip`)
struct CapSegs {
    const uint8_t* p[kMaxCapSegs];
    uint32_t len[kMaxCapSegs];
    int n = 0, idx = 0, skip = 0;
    __device__ __forceinline__ void reset(int skip_) { n = 0; idx = 0; skip = skip_; }
    __device__ __forceinline__ bool full() const { return n == kMaxCapSegs; }
    // the next `k` segments all lie before the window
    __device__ __forceinline__ bool before(unsigned long long k) const { return idx + k <= (unsigned long long)skip; }
    // l: a length word (kLenEnd, kLenWord, or a span's length, | kLenJson for one with escapes)
    __device__ __forceinline__ void push(const uint8_t* q, uint32_t l) {
        if (idx >= skip && n < kMaxCapSegs) {
            p[n] = q;
            len[n] = l;
            ++n;
        }
        ++idx;
    }
    __device__ __forceinline__ void word(unsigned long long v) { push(reinterpret_cast<const uint8_t*>(v), kLenWord); }
    __device__ __forceinline__ void bytes(Span s, bool json) {
        if (s.len > 0) push(s.p, (uint32_t)s.len | (json ? kLenJson : 0u));
    }
};

// A text: prefix (the '_' of a pair key, or none) + body (JSON-escaped when esc) + suffix (an LTSV type suffix)
struct CapText {
    Span body, suffix;
    bool us, esc;
};
// A pair: its key, its discriminant and value word, and for a string its text
struct CapPair {
    CapText key, val;
    uint32_t tag;
    unsigned long long v;
};

// One record as capnp objects: the field texts, the rows of its pairs (the first SD element's), its byte lengths
__device__ __forceinline__ uint32_t span_text_len(Span s, bool esc, bool mode2) {
    if (!esc) return (uint32_t)s.len;
    uint32_t n = 0;
    for (int k = 0; k < s.len;) {
        uint32_t w;
        n += (uint32_t)json_unescape_step(s.p, k, s.len, mode2, w);
    }
    return n;
}
__device__ __forceinline__ uint32_t text_len(const CapText& t, bool mode2) {
    return (t.us ? 1u : 0u) + span_text_len(t.body, t.esc, mode2) + (uint32_t)t.suffix.len;
}
// capnp holds a text of len bytes: its NUL included, a list of under 2^29 bytes.  Only the text counts: the span of a
// GELF string with escapes, longer than its text, has a segment length of its own.
__device__ __forceinline__ bool text_fits(uint32_t len) { return len + 1u < kCapMaxWords; }

struct CapRec {
    CapText f[CP_SDID + 1];
    uint32_t flen[CP_SDID + 1];
    uint32_t fmask;      // the field texts the Record has
    uint32_t pa, pb;     // pair rows [pa, pb)
    bool sd;             // Record.sd is Some: a pair list (possibly empty, for an RFC5424 element without pairs)
    bool mode2;          // GELF retry line: its escapes read as KeyIter's mode 2
    unsigned long long w0, w1;  // the Record's data words
};

__device__ __forceinline__ CapText plain(Span s, bool esc = false) { return CapText{s, Span{nullptr, 0}, false, esc}; }

template <class Src>
__device__ __forceinline__ void load_cap_record(const GelfEncodeParams& P, const ByteSource& B, int i, RecView& r, CapRec& c) {
    Src::load(P, B, i, r);
    if (!r.ok) return;
    const bool g = Src::kGelf;
    c.mode2 = g && (r.flags & kNlRetry) != 0u;
    uint32_t fac = kNoSeverity;
    if constexpr (!Src::kLtsv && !Src::kGelf) {
        load_msgid_facility<!Src::kOptional>(P, B, i, r);
        fac = r.facility;
    }
    c.w0 = (unsigned long long)__double_as_longlong(r.ts);
    c.w1 = fac | (r.severity << 8);
    c.fmask = 1u << CP_HOST;
    c.f[CP_HOST] = plain(r.host, g && (r.flags & kHostEsc));
    if constexpr (!Src::kOptional) {
        c.fmask |= (1u << CP_APP) | (1u << CP_PROC) | (1u << CP_MSGID);
        c.f[CP_APP] = plain(r.app);
        c.f[CP_PROC] = plain(r.proc);
        c.f[CP_MSGID] = plain(r.msgid);
    }
    if (r.msg.p) {
        c.fmask |= 1u << CP_MSG;
        c.f[CP_MSG] = plain(r.msg, g && (r.flags & kMsgEsc));
    }
    if (!g || r.full.p) {
        c.fmask |= 1u << CP_FULL;
        c.f[CP_FULL] = plain(r.full, g && (r.flags & kFullEsc));
    }
    c.sd = false;
    c.pa = c.pb = 0;
    if constexpr (Src::kSd) {
        if constexpr (Src::kLtsv || Src::kGelf) {  // one element without id, Some only with pairs
            c.sd = r.count > 0;
            c.pa = r.first;
            c.pb = r.first + r.count;
        } else if (r.count > 0) {  // RFC5424: the first element's id and its pairs, up to the next element's header
            c.sd = true;
            const uint32_t e0 = r.first;
            Span id;
            if (r.wide) id = Span{B.at(P.wentry_name[e0].x), P.wentry_name[e0].y};
            else {
                const unsigned long long v = P.entries[e0];
                id = Span{r.line + (int)(v & 0xFFFFu), (int)((v >> 16) & 0xFFFFu) - (int)(v & 0xFFFFu)};
            }
            c.fmask |= 1u << CP_SDID;
            c.f[CP_SDID] = plain(id);
            uint32_t e = e0 + 1;
            for (; e < r.first + r.count; ++e) {
                const bool hdr = r.wide ? (P.wentry_meta[e] & 0x07u) == 7u : (P.entries[e] & kE8Header) != 0ull;
                if (hdr) break;
            }
            c.pa = e0 + 1;
            c.pb = e;
        }
    }
#pragma unroll
    for (int k = 0; k <= CP_SDID; ++k) c.flen[k] = (c.fmask >> k) & 1u ? text_len(c.f[k], c.mode2) : 0u;
}

// pair row e of the record
template <class Src>
__device__ __forceinline__ void cap_pair(const GelfEncodeParams& P, const ByteSource& B, const RecView& r, uint32_t e, CapPair& q) {
    typename Src::Key k;
    typename Src::Val v;
    Src::pair(P, B, r, e, k, v);
    q.val = plain(Span{nullptr, 0});
    if constexpr (Src::kLtsv) {
        q.key = CapText{k.name, k.suffix, true, false};
        q.tag = v.tag;
        q.v = v.v;
        if (v.tag == 0u) q.val = plain(Span{B.at((int)(uint32_t)v.v), (int)(v.v >> 32)});
    } else if constexpr (Src::kGelf) {
        q.key = CapText{k.name, Span{nullptr, 0}, true, k.esc};
        q.tag = v.tag;
        q.v = v.v;
        if (v.tag == 0u) q.val = plain(Span{B.at((int)(uint32_t)v.v), (int)(v.v >> 32)}, v.esc);
    } else {
        q.key = CapText{k, Span{nullptr, 0}, true, false};
        q.tag = 0u;
        q.v = 0ull;
        q.val = plain(v);
    }
}

// output.capnp_extra pair j: static_blob holds key j at [off[2j], off[2j+1]) and its value up to off[2j+2]
__device__ __forceinline__ void cap_extra(const GelfEncodeParams& P, int j, CapPair& q) {
    const int32_t* o = P.static_key_off;
    q.key = plain(Span{P.static_blob + o[2 * j], o[2 * j + 1] - o[2 * j]});
    q.val = plain(Span{P.static_blob + o[2 * j + 1], o[2 * j + 2] - o[2 * j + 1]});
    q.tag = 0u;
    q.v = 0ull;
}

template <class Src>
__device__ __forceinline__ void any_pair(const GelfEncodeParams& P, const ByteSource& B, const RecView& r, bool extra, uint32_t j,
                                         CapPair& q) {
    if (extra) cap_extra(P, (int)j, q);
    else cap_pair<Src>(P, B, r, j, q);
}

// Places every object of the record in allocation order.  kids (optional): where the Record's 9 pointers lead.
// Returns false for a record capnp cannot hold: a text of 2^29 - 1 bytes or more, a list of 2^29 words or more.
template <class Src>
__device__ __forceinline__ bool place_all(const GelfEncodeParams& P, const ByteSource& B, const RecView& r, const CapRec& c,
                                          CapAlloc& A, CapPlace* kids) {
    bool ok = true;
    A.init();
    A.place(0, kCapRootWords);
    for (int k = 0; k <= CP_SDID; ++k) {
        if (!((c.fmask >> k) & 1u)) continue;
        ok = ok && text_fits(c.flen[k]);
        const CapPlace pl = A.place(0, cap_text_words(c.flen[k]));
        if (kids) kids[k] = pl;
    }
    for (int l = 0; l < 2; ++l) {
        const bool extra = l == 1;
        const uint32_t n = extra ? (uint32_t)P.n_static : c.pb - c.pa;
        if (extra ? n == 0u : !c.sd) continue;
        ok = ok && n < kCapMaxWords / 4u;
        const CapPlace pl = A.place(0, 1u + 4u * n);
        if (kids) kids[CP_PAIRS + l] = pl;
        for (uint32_t j = 0; j < n; ++j) {
            CapPair q;
            any_pair<Src>(P, B, r, extra, extra ? j : c.pa + j, q);
            const uint32_t kl = text_len(q.key, c.mode2);
            ok = ok && text_fits(kl);
            A.place(pl.seg, cap_text_words(kl));
            if (q.tag == 0u) {
                const uint32_t vl = text_len(q.val, c.mode2);
                ok = ok && text_fits(vl);
                A.place(pl.seg, cap_text_words(vl));
            }
        }
    }
    return ok && !A.bad;
}

// an object placed at pl, as seen from segment s: its landing pad first when it has one
__device__ __forceinline__ void pad_if_far(CapSegs& L, const CapPlace& pl, uint32_t kind, uint32_t hi) {
    if (pl.pad >= 0) L.word(cap_pad_word(kind, hi));
}
__device__ __forceinline__ void push_text(CapSegs& L, const CapText& t) {
    if (t.us) L.push(kUnderscore, 1u);
    L.bytes(t.body, t.esc);
    L.bytes(t.suffix, false);
    L.push(nullptr, kLenEnd);
}

// The segments of window L (from L.skip on, up to kMaxCapSegs of them): the segment table, then the words of each
// message segment in allocation order.  A: scratch for the layout walks.
template <class Src>
__device__ __forceinline__ void build_capnp(const GelfEncodeParams& P, const ByteSource& B, const RecView& r, const CapRec& c,
                                            CapAlloc& A, CapAlloc& A2, CapSegs& L) {
    CapPlace kids[CP_COUNT];
    place_all<Src>(P, B, r, c, A, kids);  // the segment sizes and where the Record's pointers lead
    const int nseg = A.nseg;
    for (int t = 0; t < A.table_words(); ++t) L.word(A.table_word(t));
    for (int s = 0; s < nseg && !L.full(); ++s) {
        A2.init();
        A2.place(0, kCapRootWords);
        if (s == 0) {
            L.word((unsigned long long)cap_struct_hi(2, 9) << 32);  // the root pointer: the Record right behind it
            L.word(c.w0);
            L.word(c.w1);
            for (int k = 0; k < CP_COUNT; ++k) {
                const uint32_t at = 3u + (uint32_t)k;  // the Record's pointer k
                unsigned long long w = 0ull;
                if (k <= CP_SDID) {
                    if ((c.fmask >> k) & 1u) w = cap_pointer(0, at, kids[k], 1u, cap_text_hi(c.flen[k]));
                } else if (k == CP_PAIRS ? c.sd : P.n_static > 0) {
                    w = cap_pointer(0, at, kids[k], 1u, cap_pairs_hi(k == CP_PAIRS ? c.pb - c.pa : (uint32_t)P.n_static));
                }
                L.word(w);
            }
        }
        for (int k = 0; k <= CP_SDID && !L.full(); ++k) {
            if (!((c.fmask >> k) & 1u)) continue;
            const CapPlace pl = A2.place(0, cap_text_words(c.flen[k]));
            if (pl.seg != s) continue;
            pad_if_far(L, pl, 1u, cap_text_hi(c.flen[k]));
            push_text(L, c.f[k]);
        }
        for (int l = 0; l < 2 && !L.full(); ++l) {
            const bool extra = l == 1;
            const uint32_t n = extra ? (uint32_t)P.n_static : c.pb - c.pa;
            if (extra ? n == 0u : !c.sd) continue;
            const CapPlace pl = A2.place(0, 1u + 4u * n);
            if (pl.seg == s) {
                pad_if_far(L, pl, 1u, cap_pairs_hi(n));
                L.word(cap_pairs_tag(n));
                if (L.before(4ull * n)) {
                    L.idx += 4 * (int)n;
                } else {
                    CapAlloc& K = A;  // the texts' places, one pair ahead of nothing: a copy of the walk so far
                    K = A2;
                    for (uint32_t j = 0; j < n && !L.full(); ++j) {
                        CapPair q;
                        any_pair<Src>(P, B, r, extra, extra ? j : c.pa + j, q);
                        const uint32_t at = pl.pos + 1u + 4u * j;
                        const uint32_t kl = text_len(q.key, c.mode2);
                        const CapPlace kp = K.place(pl.seg, cap_text_words(kl));
                        L.word((unsigned long long)q.tag | (q.tag == 1u && q.v ? 0x10000ull : 0ull));
                        L.word(q.tag >= 2u && q.tag <= 4u ? q.v : 0ull);
                        L.word(cap_pointer(s, at + 2u, kp, 1u, cap_text_hi(kl)));
                        unsigned long long vw = 0ull;
                        if (q.tag == 0u) {
                            const uint32_t vl = text_len(q.val, c.mode2);
                            vw = cap_pointer(s, at + 3u, K.place(pl.seg, cap_text_words(vl)), 1u, cap_text_hi(vl));
                        }
                        L.word(vw);
                    }
                }
            }
            for (uint32_t j = 0; j < n && !L.full(); ++j) {
                CapPair q;
                any_pair<Src>(P, B, r, extra, extra ? j : c.pa + j, q);
                const uint32_t kl = text_len(q.key, c.mode2);
                const CapPlace kp = A2.place(pl.seg, cap_text_words(kl));
                if (kp.seg == s) {
                    pad_if_far(L, kp, 1u, cap_text_hi(kl));
                    push_text(L, q.key);
                }
                if (q.tag == 0u) {
                    const uint32_t vl = text_len(q.val, c.mode2);
                    const CapPlace vp = A2.place(pl.seg, cap_text_words(vl));
                    if (vp.seg == s) {
                        pad_if_far(L, vp, 1u, cap_text_hi(vl));
                        push_text(L, q.val);
                    }
                }
            }
        }
    }
}

// The warp-uniform byte loop over the segments of every lane's record (`live` = this lane has one).  `done` = bytes of
// the record written before this window (a CK_END pads to the next multiple of 8).  kJson: the list may hold GELF spans
// with JSON escapes (only FromGelf instantiates it).
template <bool kJson, class Sink>
__device__ __forceinline__ void run_capnp(const CapSegs& L, bool live, Sink& s, bool mode2, unsigned long long& done) {
    int si = 0, k = 0, len = 0;
    uint32_t kind = CK_WORD;
    const uint8_t* p = nullptr;
    bool more = live && L.n > 0;
    auto enter = [&](int j) {
        p = L.p[j];
        const uint32_t l = L.len[j];
        kind = l == kLenWord ? CK_WORD : l == kLenEnd ? CK_END : (l & kLenJson) ? CK_JSON : CK_RAW;
        len = kind == CK_WORD ? 8 : kind == CK_END ? 8 - (int)(done & 7u) : (int)(l & ~kLenJson);
        k = 0;
    };
    if (more) enter(0);
    while (__any_sync(0xFFFFFFFFu, more)) {
        if (more) {
            uint32_t w = 0;
            int n = 4;
            if (kind == CK_WORD) {
                w = (uint32_t)(reinterpret_cast<unsigned long long>(p) >> (8 * k));
                k += 4;
            } else if (kind == CK_END) {
                if (k + 4 > len) n = 1;
                k += n;
            } else {
                w = p[k];
                if (k + 4 <= len) w |= ((uint32_t)p[k + 1] << 8) | ((uint32_t)p[k + 2] << 16) | ((uint32_t)p[k + 3] << 24);
                else n = 1;
                if (kJson && kind == CK_JSON && (n == 1 || ((w & 0xFFu) == 0x5Cu) || ((w >> 8 & 0xFFu) == 0x5Cu) ||
                                                 ((w >> 16 & 0xFFu) == 0x5Cu) || ((w >> 24) == 0x5Cu))) {
                    n = json_unescape_step(p, k, len, mode2, w);  // one escape (or byte) unescaped
                } else {
                    k += n;
                }
            }
            s.push(w, n);
            done += (unsigned)n;
            if (k >= len) {  // next segment (none is empty)
                if (++si < L.n) enter(si);
                else more = false;
            }
        }
    }
}

template <class Src, class Sink>
__device__ __forceinline__ void emit_capnp(const GelfEncodeParams& P, const ByteSource& B, const RecView& r, const CapRec& c, bool live,
                                           Sink& s) {
    CapSegs L;
    CapAlloc A, A2;
    unsigned long long done = 0;
    int skip = 0;
    for (;;) {
        L.reset(skip);
        if (live) build_capnp<Src>(P, B, r, c, A, A2, L);
        run_capnp<Src::kGelf>(L, live, s, c.mode2, done);
        skip += kMaxCapSegs;
        if (!__any_sync(0xFFFFFFFFu, live && L.full())) break;
    }
    if (live) s.finish();
}

template <class Src>
__global__ void __launch_bounds__(kEncLines) capnp_size_kernel(const __grid_constant__ GelfEncodeParams P) {
    extern __shared__ __align__(128) uint8_t tile[];
    __shared__ __align__(8) EncShared sh;
    if (*P.bad_offsets) return;
    const int first = blockIdx.x * kEncLines, last = min(P.n, first + kEncLines);
    const ByteSource B = stage_lines(P, tile, &sh.mbar, first, last);
    const int i = sorted_line(P, sh, first, last);
    if (i < 0) return;
    RecView r;
    CapRec c;
    r.ok = false;
    load_cap_record<Src>(P, B, i, r, c);
    unsigned long long len = 0;
    if (r.ok) {
        CapAlloc A;
        if (place_all<Src>(P, B, r, c, A, nullptr)) len = framed_len(A.bytes(), P.out_framing);
        else atomicMin(P.long_json_span, (uint32_t)P.offsets[i]);  // refused: the call fails, nothing is written
    }
    P.lens[i] = len;
    P.status[i] = (uint8_t)Src::status(P, i);
    if constexpr (Src::kLtsv) P.ltsv_stop[i] = ltsv_stop(P, i);
}

template <class Src>
__global__ void __launch_bounds__(kEncLines) capnp_write_kernel(const __grid_constant__ GelfEncodeParams P) {
    extern __shared__ __align__(128) uint8_t tile[];
    __shared__ __align__(8) EncShared sh;
    if (*P.bad_offsets) return;
    const int first = blockIdx.x * kEncLines, last = min(P.n, first + kEncLines);
    if (P.out_framing != kOutNone && first + (int)threadIdx.x < last) {
        // output.framing of line first + tid, stored before any record of the CTA is emitted (see gelf_write_kernel)
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
    CapRec c;
    r.ok = false;
    c.mode2 = false;
    if (live) load_cap_record<Src>(P, B, i, r, c);
    WordSink s(P.out + at + (live && P.out_framing == kOutSyslen ? sh.pre[i - first] : 0));
    emit_capnp<Src>(P, B, r, c, live && r.ok, s);
}

template <class Src>
cudaError_t configure_capnp_src(int max_tile_bytes) {
    return configure_passes(capnp_size_kernel<Src>, capnp_write_kernel<Src>, max_tile_bytes);
}

template <class Src>
cudaError_t launch_capnp_src(const GelfEncodeParams& p, void* d_scan_temp, size_t scan_temp_bytes, cudaStream_t stream) {
    return launch_passes(capnp_size_kernel<Src>, capnp_write_kernel<Src>, p, d_scan_temp, scan_temp_bytes, stream);
}

}  // namespace

cudaError_t configure_capnp_encode(int max_tile_bytes) {
    cudaError_t e = configure_capnp_src<From5424>(max_tile_bytes);
    if (e != cudaSuccess) return e;
    e = configure_capnp_src<From3164>(max_tile_bytes);
    if (e != cudaSuccess) return e;
    e = configure_capnp_src<FromLtsv>(max_tile_bytes);
    if (e != cudaSuccess) return e;
    return configure_capnp_src<FromGelf>(max_tile_bytes);
}

cudaError_t launch_capnp_encode(int fmt, const GelfEncodeParams& p, void* d_scan_temp, size_t scan_temp_bytes, cudaStream_t stream) {
    if (p.n <= 0) return cudaSuccess;
    switch (fmt) {
        case 0: return launch_capnp_src<From5424>(p, d_scan_temp, scan_temp_bytes, stream);
        case 1: return launch_capnp_src<FromLtsv>(p, d_scan_temp, scan_temp_bytes, stream);
        case 2: return launch_capnp_src<FromGelf>(p, d_scan_temp, scan_temp_bytes, stream);
        case 3: return launch_capnp_src<From3164>(p, d_scan_temp, scan_temp_bytes, stream);
        default: return cudaErrorInvalidValue;
    }
}

}  // namespace fg
