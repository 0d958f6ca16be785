// fg_ltsv_encode.cu — the LTSV encoder fused after the decoder on the device: Record -> LTSV text (output.format = "ltsv").
//
// H100-native replacement for LTSVEncoder::encode (flowgger src/flowgger/encoder/ltsv_encoder.rs:66-123).  The record is
// written field by field in Record order, with no sorting and no de-duplication (a repeated key is written twice):
//   1. every pair of every SD element, its name without one leading '_' (every decoder's names have one:
//      rfc5424_decoder.rs:220-222 adds it, ltsv_decoder.rs:128-181 writes '_' + name + suffix, gelf_decoder.rs:99-104
//      keeps or adds it), the sd_id ignored;
//   2. output.ltsv_extra: one literal composed on the host (fg_set_ltsv_extra: sorted, '_' stripped, already escaped);
//   3. host (as it is, "host:" when empty) and time (Record.ts, Display for f64: fg_ftoa.cuh);
//   4. message, full_message, level, facility, appname, procid, msgid, each only when the Record has it.
// Fields are separated by '\t'; keys and values go through LTSVString::insert's replacements (fg_ltsv_text.cuh).  A typed
// value is written as Rust's to_string: true / false, Display for f64, decimal I64 / U64; Null as "".
//
// The record view, the sinks, the CTA staging in order of line length and the launch sequence are the GELF encoder's
// (fg_encode_view.cuh); only the text differs.  A record becomes a flat list of segments (pointer, length, kind) and all
// lanes of a warp then run one byte loop over their lists: four bytes per iteration for text (the replacements keep
// every byte one byte, so they are applied to the word), one unescape step for a GELF span that holds JSON escapes, one
// byte for a number, whose text is laid out by fg_ftoa.cuh as digits plus a run of zeros.
#include "fg_encode_view.cuh"
#include "fg_ftoa.cuh"
#include "fg_ltsv_text.cuh"
#include "fg_out_frame.cuh"

namespace fg {

namespace {

// the kind of a segment, in bits 29..31 of its length
enum : uint32_t { SK_RAW = 0, SK_VAL = 1, SK_KEY = 2, SK_JSON_VAL = 3, SK_JSON_KEY = 4, SK_NUM = 5 };
constexpr int kKindShift = 29;
constexpr int kLenMask = (1 << kKindShift) - 1;

__device__ const uint8_t kLtsvLit[] = "\t:\thost:\ttime:\tmessage:\tfull_message:\tlevel:\tfacility:\tappname:\tprocid:\tmsgid:01234567";
enum { LT_TAB = 0, LT_COLON = 1, LT_HOST = 2, LT_TIME = 8, LT_MESSAGE = 14, LT_FULL = 23, LT_LEVEL = 37, LT_FACILITY = 44,
       LT_APPNAME = 54, LT_PROCID = 63, LT_MSGID = 71, LT_DIGITS = 78 };

// a number segment: the 8 value bytes themselves stand in the pointer, its fg_tag in the length
constexpr uint32_t kTagFacility = 4u;  // Record.facility (u8) is written as a U64

constexpr int kMaxLtsvSegs = 56;  // a record with more segments is emitted in several windows (rebuilt with `skip`)
struct LtsvSegs {
    const uint8_t* p[kMaxLtsvSegs];
    uint32_t len[kMaxLtsvSegs];
    int n = 0, idx = 0, skip = 0;
    bool first = true;  // no field written yet: the next one gets no '\t'
    __device__ __forceinline__ void reset(int skip_) { n = 0; idx = 0; skip = skip_; first = true; }
    __device__ __forceinline__ void push(const uint8_t* q, int l, uint32_t kind) {
        if (l <= 0) return;
        if (idx >= skip && n < kMaxLtsvSegs) {
            p[n] = q;
            len[n] = (uint32_t)l | (kind << kKindShift);
            ++n;
        }
        ++idx;
    }
    // a span of text: one longer than the length field is cut into several segments, which is exact because the
    // replacements are per byte.  A span with JSON escapes is not cut (a cut could split an escape): the size kernel
    // fails the call for one that long (long_json_span_kernel), and its record stays inside the span.
    __device__ __forceinline__ void span(const uint8_t* q, int l, uint32_t kind) {
        if (kind < SK_JSON_VAL)
            for (; l > kLenMask; q += kLenMask, l -= kLenMask) push(q, kLenMask, kind);
        else
            l &= kLenMask;
        push(q, l, kind);
    }
    __device__ __forceinline__ void lit(int at, int l) { push(kLtsvLit + at, l, SK_RAW); }
    // `\tname:` of a fixed field, the tab dropped for the record's first field
    __device__ __forceinline__ void field(int at, int l) {
        lit(at + (first ? 1 : 0), l - (first ? 1 : 0));
        first = false;
    }
    __device__ __forceinline__ void key_start() {
        if (!first) lit(LT_TAB, 1);
        first = false;
    }
    __device__ __forceinline__ void num(unsigned long long v, uint32_t tag) {
        push(reinterpret_cast<const uint8_t*>(v), (int)tag, SK_NUM);
    }
    __device__ __forceinline__ void text(Span s, bool json) { span(s.p, s.len, json ? SK_JSON_VAL : SK_VAL); }
};

// one SD pair of the record
template <class Src>
__device__ __forceinline__ void ltsv_pair(const GelfEncodeParams& P, const ByteSource& B, const RecView& r, uint32_t e, LtsvSegs& L) {
    typename Src::Key k;
    typename Src::Val v;
    if (!Src::pair(P, B, r, e, k, v)) return;  // an RFC5424 element header
    L.key_start();
    if constexpr (Src::kLtsv) {  // '_' + name + suffix: the name and the type's suffix
        L.span(k.name.p, k.name.len, SK_KEY);
        L.push(k.suffix.p, k.suffix.len, SK_KEY);
        L.lit(LT_COLON, 1);
        if (v.tag == 0u) L.span(B.at((int)(uint32_t)v.v), (int)(v.v >> 32), SK_VAL);
        else L.num(v.v, v.tag);
    } else if constexpr (Src::kGelf) {  // the name without its '_' (load_pair_gelf), strings as their unescaped text
        L.span(k.name.p, k.name.len, k.esc ? SK_JSON_KEY : SK_KEY);
        L.lit(LT_COLON, 1);
        if (v.tag == 0u) L.span(B.at((int)(uint32_t)v.v), (int)(v.v >> 32), v.esc ? SK_JSON_VAL : SK_VAL);
        else if (v.tag != 5u) L.num(v.v, v.tag);  // Null: ""
    } else {  // RFC5424: the name as written (the decoder's '_' is the one stripped)
        L.span(k.p, k.len, SK_KEY);
        L.lit(LT_COLON, 1);
        L.span(v.p, v.len, SK_VAL);
    }
}

template <class Src>
__device__ __forceinline__ void build_ltsv(const GelfEncodeParams& P, const ByteSource& B, const RecView& r, LtsvSegs& L) {
    if constexpr (Src::kSd)
        for (uint32_t e = r.first; e < r.first + r.count; ++e) ltsv_pair<Src>(P, B, r, e, L);
    if (P.n_static > 0) {  // output.ltsv_extra: `\tkey:value` per extra
        L.span(P.static_blob + (L.first ? 1 : 0), P.n_static - (L.first ? 1 : 0), SK_RAW);
        L.first = false;
    }
    const bool g = Src::kGelf;
    L.field(LT_HOST, 6);
    L.text(r.host, g && (r.flags & kHostEsc));
    L.field(LT_TIME, 6);
    L.num((unsigned long long)__double_as_longlong(r.ts), 2u);
    if (r.msg.p) {
        L.field(LT_MESSAGE, 9);
        L.text(r.msg, g && (r.flags & kMsgEsc));
    }
    if (!g || r.full.p) {
        L.field(LT_FULL, 14);
        L.text(r.full, g && (r.flags & kFullEsc));
    }
    if (r.severity != kNoSeverity) {
        L.field(LT_LEVEL, 7);
        L.lit(LT_DIGITS + (int)(r.severity & 7u), 1);
    }
    if constexpr (!Src::kLtsv && !Src::kGelf) {  // RFC5424 and RFC3164 carry the facility (None without <PRI>)
        if (r.facility != kNoSeverity) {
            L.field(LT_FACILITY, 10);
            L.num(r.facility, kTagFacility);
        }
    }
    if constexpr (!Src::kOptional) {  // RFC5424: appname, procid and msgid are always Some
        L.field(LT_APPNAME, 9);
        L.text(r.app, false);
        L.field(LT_PROCID, 8);
        L.text(r.proc, false);
        L.field(LT_MSGID, 7);
        L.text(r.msgid, false);
    }
}

// the row of line i, with msgid and facility where the source has them
template <class Src>
__device__ __forceinline__ void load_record(const GelfEncodeParams& P, const ByteSource& B, int i, RecView& r) {
    Src::load(P, B, i, r);
    if constexpr (!Src::kLtsv && !Src::kGelf)
        if (r.ok) load_msgid_facility<!Src::kOptional>(P, B, i, r);
}

// the text of a number segment
__device__ __forceinline__ void number_text(unsigned long long v, uint32_t tag, FtoaText& t) {
    if (tag == 1u) {  // "true" / "false"
        ftoa_word(t, v ? 0x65757274u : 0x736C6166u, 4);
        t.buf[4] = 'e';
        t.blen = t.zpos = v ? 4 : 5;
    } else if (tag == 2u) {
        f64_display(__longlong_as_double((long long)v), t);
    } else {
        int_display(v, tag == 3u, t);
    }
}

// The warp-uniform byte loop over the segments of every lane's record (`live` = this lane has one).  kJson: the list may
// hold GELF spans with JSON escapes (only FromGelf instantiates it).
template <bool kJson, class Sink>
__device__ __forceinline__ void run_ltsv(const LtsvSegs& L, bool live, Sink& s, bool mode2) {
    int si = 0, k = 0, len = 0;
    uint32_t kind = SK_RAW;
    const uint8_t* p = nullptr;
    FtoaText num;
    bool more = live && L.n > 0;
    auto enter = [&](int j) {
        p = L.p[j];
        kind = L.len[j] >> kKindShift;
        len = (int)(L.len[j] & kLenMask);
        k = 0;
        if (kind == SK_NUM) {
            number_text(reinterpret_cast<unsigned long long>(p), (uint32_t)len, num);
            len = num.len();
        }
    };
    if (more) enter(0);
    while (__any_sync(0xFFFFFFFFu, more)) {
        if (more) {
            uint32_t w;
            int n = 1;
            if (kind == SK_NUM) {
                w = num.at(k);
                k += 1;
            } else {
                const bool key = kind == SK_KEY || kind == SK_JSON_KEY;
                w = p[k];
                if (k + 4 <= len) {
                    w |= ((uint32_t)p[k + 1] << 8) | ((uint32_t)p[k + 2] << 16) | ((uint32_t)p[k + 3] << 24);
                    n = 4;
                }
                if (kJson && kind >= SK_JSON_VAL && (n == 1 || ltsv_eq4(w, 0x5C5C5C5Cu))) {  // one escape (or byte) unescaped
                    n = json_unescape_step(p, k, len, mode2, w);
                } else {
                    k += n;
                }
                if (kind != SK_RAW) w = ltsv_escape4(w, key);
            }
            s.push(w, n);
            if (k >= len) {  // next segment (none is empty)
                if (++si < L.n) enter(si);
                else more = false;
            }
        }
    }
}

template <class Src, class Sink>
__device__ __forceinline__ void emit_ltsv(const GelfEncodeParams& P, const ByteSource& B, const RecView& r, bool live, Sink& s) {
    LtsvSegs L;
    int skip = 0;
    for (;;) {
        L.reset(skip);
        if (live) build_ltsv<Src>(P, B, r, L);
        run_ltsv<Src::kGelf>(L, live, s, Src::kGelf && (r.flags & kNlRetry) != 0u);
        skip += kMaxLtsvSegs;
        if (!__any_sync(0xFFFFFFFFu, live && L.idx > skip)) break;
    }
    if (live) s.finish();
}

template <class Src>
__global__ void __launch_bounds__(kEncLines) ltsv_size_kernel(const __grid_constant__ GelfEncodeParams P) {
    extern __shared__ __align__(128) uint8_t tile[];
    __shared__ __align__(8) EncShared sh;
    if (*P.bad_offsets) return;
    const int first = blockIdx.x * kEncLines, last = min(P.n, first + kEncLines);
    const ByteSource B = stage_lines(P, tile, &sh.mbar, first, last);
    const int i = sorted_line(P, sh, first, last);
    const bool valid = i >= 0;
    RecView r;
    r.ok = false;
    if (valid) load_record<Src>(P, B, i, r);
    CountSink s;
    emit_ltsv<Src>(P, B, r, r.ok, s);
    if (!valid) return;
    P.lens[i] = r.ok ? framed_len(s.n, P.out_framing) : 0ull;
    P.status[i] = (uint8_t)Src::status(P, i);
    if constexpr (Src::kLtsv) P.ltsv_stop[i] = ltsv_stop(P, i);
}

template <class Src>
__global__ void __launch_bounds__(kEncLines) ltsv_write_kernel(const __grid_constant__ GelfEncodeParams P) {
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
    r.ok = false;
    if (live) load_record<Src>(P, B, i, r);
    WordSink s(P.out + at + (live && P.out_framing == kOutSyslen ? sh.pre[i - first] : 0));
    emit_ltsv<Src>(P, B, r, live && r.ok, s);
}

template <class Src>
cudaError_t configure_ltsv_src(int max_tile_bytes) {
    return configure_passes(ltsv_size_kernel<Src>, ltsv_write_kernel<Src>, max_tile_bytes);
}

template <class Src>
cudaError_t launch_ltsv_src(const GelfEncodeParams& p, void* d_scan_temp, size_t scan_temp_bytes, cudaStream_t stream) {
    return launch_passes(ltsv_size_kernel<Src>, ltsv_write_kernel<Src>, p, d_scan_temp, scan_temp_bytes, stream);
}

}  // namespace

cudaError_t configure_ltsv_encode(int max_tile_bytes) {
    cudaError_t e = configure_ltsv_src<From5424>(max_tile_bytes);
    if (e != cudaSuccess) return e;
    e = configure_ltsv_src<From3164>(max_tile_bytes);
    if (e != cudaSuccess) return e;
    e = configure_ltsv_src<FromLtsv>(max_tile_bytes);
    if (e != cudaSuccess) return e;
    return configure_ltsv_src<FromGelf>(max_tile_bytes);
}

cudaError_t launch_ltsv_encode(int fmt, const GelfEncodeParams& p, void* d_scan_temp, size_t scan_temp_bytes, cudaStream_t stream) {
    if (p.n <= 0) return cudaSuccess;
    switch (fmt) {
        case 0: return launch_ltsv_src<From5424>(p, d_scan_temp, scan_temp_bytes, stream);
        case 1: return launch_ltsv_src<FromLtsv>(p, d_scan_temp, scan_temp_bytes, stream);
        case 2:
            if (p.long_json_span) long_json_span_kernel<<<(p.n + kEncLines - 1) / kEncLines, kEncLines, 0, stream>>>(p, kLenMask);
            return launch_ltsv_src<FromGelf>(p, d_scan_temp, scan_temp_bytes, stream);
        case 3: return launch_ltsv_src<From3164>(p, d_scan_temp, scan_temp_bytes, stream);
        default: return cudaErrorInvalidValue;
    }
}

}  // namespace fg
