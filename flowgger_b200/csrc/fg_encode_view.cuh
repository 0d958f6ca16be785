// fg_encode_view.cuh — what the fused encoders (fg_gelf_encode.cu: GELF, fg_ltsv_encode.cu: LTSV) read and how they
// write: the record view of each decoder's device-resident results (RecView, load_view*, load_pair*, the four record
// sources), the counting and writing sinks, and the staging of a CTA's 256 lines in shared memory in order of line
// length.  The two encoders differ only in the text they emit for a record.
#pragma once
#include <cub/device/device_scan.cuh>

#include "fg_kernels.cuh"

#include "fg_common.cuh"
#include "fg_gelf.cuh"
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

// An LTSV or GELF record's sink: the extent of the side table's value column, which tells the byte loop the number segments
template <class Sink>
struct NumSink {
    Sink& s;
    const unsigned long long* vals;
    uint32_t cap;
    __device__ __forceinline__ void push(uint32_t w, int k) { s.push(w, k); }
};
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
    uint32_t flags;                    // GELF: the row's FG_FLAG_* (escaped spans, retry line)
    // read by the LTSV encoder only (GELF writes neither), so loaded apart (load_msgid_facility): Record.msgid (RFC5424)
    // and Record.facility (0xFF: None)
    Span msgid;
    uint32_t facility;
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

// Record.msgid and Record.facility of a loaded RFC5424 or RFC3164 row (LTSV and GELF rows have neither).  Kept out of
// load_view / load_view_3164: loading them there moves the GELF kernels' register allocation.
template <bool k5424>
__device__ __forceinline__ void load_msgid_facility(const GelfEncodeParams& P, const ByteSource& B, int i, RecView& r) {
    if constexpr (k5424) {
        const uint4 lo4 = P.rows[2 * (size_t)i], hi4 = P.rows[2 * (size_t)i + 1];
        r.facility = (lo4.z >> 8) & 0xFFu;
        if (r.wide) {
            const int2 m = P.wide_rows[lo4.w].msgid;
            r.msgid = Span{B.at(m.x), m.y};
        } else {
            const int sp4 = (int)(hi4.z & 0xFFFFu), sp5 = (int)(hi4.z >> 16);
            r.msgid = Span{r.line + sp4 + 1, sp5 - sp4 - 1};
        }
    } else {
        r.facility = (P.col_meta[i] >> 8) & 0xFFu;
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

// A GELF row (fg_parse_gelf.cu): the column layout of LTSV.  msg.x < 0 / full.x < 0: the object has no short_message /
// full_message (None); a row without "timestamp" (FG_FLAG_TS_MISSING) takes the call's wall clock.
constexpr uint32_t kTsMissing = 0x01u, kHostEsc = 0x04u, kMsgEsc = 0x08u, kFullEsc = 0x10u, kNlRetry = 0x20u;  // FG_FLAG_*
__device__ __forceinline__ void load_view_gelf(const GelfEncodeParams& P, const ByteSource& B, int i, RecView& r) {
    const uint32_t meta = P.col_meta[i];
    r.ok = (meta & 0xFFu) == 0u;
    r.wide = false;
    r.has_sd = false;
    r.first = r.count = 0;
    if (!r.ok) return;
    r.severity = (meta >> 16) & 0xFFu;
    r.flags = meta >> 24;
    r.ts = (r.flags & kTsMissing) ? P.gelf_now : P.col_ts[i];
    const int2 h = P.col_host[i], m = P.col_msg[i], f = P.col_full[i], sd = P.col_sd[i];
    r.host = Span{B.at(h.x), h.y};
    r.msg = m.x >= 0 ? Span{B.at(m.x), m.y} : Span{nullptr, 0};
    r.full = f.x >= 0 ? Span{B.at(f.x), f.y} : Span{nullptr, 0};
    r.first = (uint32_t)sd.x;
    r.count = (uint32_t)sd.y;
    // an overflowed side table (the batch is redone) leaves rows whose range names other lines' rows: read none
    if ((unsigned long long)r.first + r.count > (unsigned long long)P.wentry_cap || *P.gelf_entries > P.wentry_cap) r.ok = false;
}

// A GELF member.  Its key after the '_' is the name, or the name without its leading '_' (FG_EM_NO_PREFIX,
// gelf_decoder.rs:99-103); `name` is that raw span.  esc: the span holds JSON escapes (FG_EM_NAME_ESC), so its bytes are
// read through KeyIter; plain names are compared byte by byte.  A value is a string span (tag 0; esc = FG_EM_UNESCAPE)
// or the fg_tag of its 8 value bytes.
struct GelfKey {
    Span name;
    bool esc, mode2;
};
struct GelfVal {
    unsigned long long v;
    uint32_t tag;
    uint32_t e;  // its row
    bool esc;
};
constexpr uint32_t kEmUnescape = 0x08u, kEmNoPrefix = 0x10u, kEmNameEsc = 0x40u;  // FG_EM_*

__device__ __forceinline__ bool load_pair_gelf(const GelfEncodeParams& P, const ByteSource& B, const RecView& r, uint32_t e, GelfKey& key,
                                               GelfVal& val) {
    const uint32_t m = P.wentry_meta[e];
    const int2 nm = P.wentry_name[e];
    key.name = Span{B.at(nm.x), nm.y};
    key.esc = (m & kEmNameEsc) != 0u;
    key.mode2 = (r.flags & kNlRetry) != 0u;
    if (m & kEmNoPrefix) {  // drop the '_' the name starts with: one raw byte, or the escape that spells it
        int k = 1;
        if (key.esc) {
            KeyIter it;
            key_iter_init(it, key.name.p, 0, key.name.len, key.mode2);
            key_iter_next(it);
            k = it.i;
        }
        key.name.p += k;
        key.name.len -= k;
    }
    val.v = P.wentry_val[e];
    val.tag = m & 0x07u;
    val.e = e;
    val.esc = (m & kEmUnescape) != 0u;
    return true;
}

// Whether a GELF row holds a span with JSON escapes longer than `limit` bytes, the longest span an encoder's segment
// length field holds.  Such a span is not cut into segments (a cut could split an escape): long_json_span_kernel flags
// it and the call fails.  A member name is measured with the '_' load_pair_gelf strips (one byte, or the six of
// \u005f): a name up to six bytes shorter than the limit is refused too, which errs on the safe side.
__device__ __forceinline__ bool json_span_over(const GelfEncodeParams& P, const RecView& r, int limit) {
    if (((r.flags & kHostEsc) && r.host.len > limit) || ((r.flags & kMsgEsc) && r.msg.len > limit) ||
        ((r.flags & kFullEsc) && r.full.len > limit))
        return true;
    for (uint32_t e = r.first; e < r.first + r.count; ++e) {
        const uint32_t m = P.wentry_meta[e];
        if ((m & kEmNameEsc) && P.wentry_name[e].y > limit) return true;
        if ((m & 0x07u) == 0u && (m & kEmUnescape) && (int)(P.wentry_val[e] >> 32) > limit) return true;
    }
    return false;
}

// GELF source: sets *P.long_json_span when a line holds a span json_span_over finds.  Only a line longer than `limit`
// can hold one, so the launchers run this kernel, one thread per line, only for a context whose lines may be that long
// (fg_abi.cu sets P.long_json_span then), and the size and write kernels carry no code for it.
__global__ void long_json_span_kernel(const __grid_constant__ GelfEncodeParams P, int limit) {
    const int i = blockIdx.x * blockDim.x + (int)threadIdx.x;
    if (*P.bad_offsets || i >= P.n || P.offsets[i + 1] - P.offsets[i] <= limit) return;
    RecView r;
    load_view_gelf(P, ByteSource{P.bytes, 0}, i, r);
    if (r.ok && json_span_over(P, r, limit)) *P.long_json_span = 1u;
}

// The record sources the kernels are instantiated for.  kSd: the record may carry structured data.  kOptional:
// application_name and process_id are None, and level is None without a severity.  kLtsv: pairs are LtsvKey / LtsvVal
// (composed keys, typed values), and the size pass writes the "Missing value" stop of every line.  kGelf: pairs are
// GelfKey / GelfVal, full_message may be None, and spans may hold JSON escapes.  kWriteCtas: the CTAs per SM
// gelf_write_kernel is allocated for (launch bounds; 0: ptxas's choice).  It holds each write kernel at the registers it
// had before the output.framing code was added to it (From3164 48, FromGelf 64): without the bound, ptxas cut FromGelf to
// 48 registers with 214 B of spill stores, 3-4 % slower on the GELF workload.  The LTSV encoder's kernels
// (fg_ltsv_encode.cu) have no such bound; ptxas (CUDA 12.9, sm_90a) gives its size kernels 64 / 48 / 48 / 48 registers
// and its write kernels 64 / 62 / 64 / 48 (From5424 / From3164 / FromLtsv / FromGelf), with spill stores only for
// FromGelf (50 B size, 52 B write).
struct From5424 {
    static constexpr bool kSd = true, kOptional = false, kLtsv = false, kGelf = false;
    static constexpr int kWriteCtas = 0;
    using Key = Span;
    using Val = Span;
    static __device__ __forceinline__ void load(const GelfEncodeParams& P, const ByteSource& B, int i, RecView& r) { load_view(P, B, i, r); }
    static __device__ __forceinline__ uint32_t status(const GelfEncodeParams& P, int i) { return P.rows[2 * (size_t)i].z & 0xFFu; }
    static __device__ __forceinline__ bool pair(const GelfEncodeParams& P, const ByteSource& B, const RecView& r, uint32_t e, Key& k, Val& v) {
        return load_pair(P, B, r, e, k, v);
    }
};
struct From3164 {
    static constexpr bool kSd = false, kOptional = true, kLtsv = false, kGelf = false;
    static constexpr int kWriteCtas = 5;
    using Key = Span;
    using Val = Span;
    static __device__ __forceinline__ void load(const GelfEncodeParams& P, const ByteSource& B, int i, RecView& r) { load_view_3164(P, B, i, r); }
    static __device__ __forceinline__ uint32_t status(const GelfEncodeParams& P, int i) { return P.col_meta[i] & 0xFFu; }
    static __device__ __forceinline__ bool pair(const GelfEncodeParams& P, const ByteSource& B, const RecView& r, uint32_t e, Key& k, Val& v) {
        return load_pair(P, B, r, e, k, v);
    }
};
struct FromLtsv {
    static constexpr bool kSd = true, kOptional = true, kLtsv = true, kGelf = false;
    static constexpr int kWriteCtas = 0;
    using Key = LtsvKey;
    using Val = LtsvVal;
    static __device__ __forceinline__ void load(const GelfEncodeParams& P, const ByteSource& B, int i, RecView& r) { load_view_ltsv(P, B, i, r); }
    static __device__ __forceinline__ uint32_t status(const GelfEncodeParams& P, int i) { return P.col_meta[i] & 0xFFu; }
    static __device__ __forceinline__ bool pair(const GelfEncodeParams& P, const ByteSource& B, const RecView&, uint32_t e, Key& k, Val& v) {
        return load_pair_ltsv(P, B, e, k, v);
    }
};
struct FromGelf {
    static constexpr bool kSd = true, kOptional = true, kLtsv = false, kGelf = true;
    static constexpr int kWriteCtas = 4;
    using Key = GelfKey;
    using Val = GelfVal;
    static __device__ __forceinline__ void load(const GelfEncodeParams& P, const ByteSource& B, int i, RecView& r) { load_view_gelf(P, B, i, r); }
    static __device__ __forceinline__ uint32_t status(const GelfEncodeParams& P, int i) { return P.col_meta[i] & 0xFFu; }
    static __device__ __forceinline__ bool pair(const GelfEncodeParams& P, const ByteSource& B, const RecView& r, uint32_t e, Key& k, Val& v) {
        return load_pair_gelf(P, B, r, e, k, v);
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
    uint8_t pre[kEncLines];  // write kernel, syslen: prefix length of each line of the CTA
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

// chunk totals: base[k + 1] = base[k] + bytes of this chunk (one thread)
__global__ void gelf_base_kernel(const __grid_constant__ GelfEncodeParams P) {
    if (*P.bad_offsets) return;
    const unsigned long long total = P.rel[P.n - 1] + P.lens[P.n - 1];
    P.base[1] = P.base[0] + total;
}

using EncodeKernel = void (*)(const GelfEncodeParams);

cudaError_t configure_passes(EncodeKernel size_k, EncodeKernel write_k, int max_tile_bytes) {
    cudaError_t e = cudaFuncSetAttribute(size_k, cudaFuncAttributeMaxDynamicSharedMemorySize, max_tile_bytes);
    if (e != cudaSuccess) return e;
    return cudaFuncSetAttribute(write_k, cudaFuncAttributeMaxDynamicSharedMemorySize, max_tile_bytes);
}

// size pass, exclusive sum of the record lengths, this launch's base, write pass
cudaError_t launch_passes(EncodeKernel size_k, EncodeKernel write_k, const GelfEncodeParams& p, void* d_scan_temp, size_t scan_temp_bytes,
                          cudaStream_t stream) {
    const int grid = (p.n + kEncLines - 1) / kEncLines;
    size_k<<<grid, kEncLines, p.tile_bytes, stream>>>(p);
    cudaError_t e = cub::DeviceScan::ExclusiveSum(d_scan_temp, scan_temp_bytes, p.lens, p.rel, p.n, stream);
    if (e != cudaSuccess) return e;
    gelf_base_kernel<<<1, 1, 0, stream>>>(p);
    write_k<<<grid, kEncLines, p.tile_bytes, stream>>>(p);
    return cudaGetLastError();
}

}  // namespace

}  // namespace fg
