// flowgger.cpp — host-side mirror of the reference's decoder-facing interface (see flowgger.hpp).
// No parsing happens here: spans and scalars come from the CUDA kernels through the C ABI; this
// file only copies them into owned Records (applying the deferred unescapes) and frames batches.
#include "flowgger.hpp"

#include <algorithm>
#include <cinttypes>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <istream>
#include <mutex>
#include <ostream>
#include <sstream>
#include <stdexcept>
#include <thread>

namespace flowgger {

// ---------------------------------------------------------------------------
// small string helpers
// ---------------------------------------------------------------------------
static std::string lower(std::string s) {
    for (auto& c : s)
        if (c >= 'A' && c <= 'Z') c = (char)(c + 32);
    return s;
}

static int ltsv_type_of(const std::string& t) {
    const std::string l = lower(t);
    if (l == "string") return FG_LTSV_STRING;
    if (l == "bool") return FG_LTSV_BOOL;
    if (l == "f64") return FG_LTSV_F64;
    if (l == "i64") return FG_LTSV_I64;
    if (l == "u64") return FG_LTSV_U64;
    return -1;
}

// Unicode White_Space (str::trim), same table as the kernels use
static size_t ws_front(std::string_view s) {
    if (s.empty()) return 0;
    const unsigned char c0 = (unsigned char)s[0];
    if ((c0 >= 9 && c0 <= 13) || c0 == 32) return 1;
    if (s.size() >= 2 && c0 == 0xC2) {
        const unsigned char c1 = (unsigned char)s[1];
        return (c1 == 0x85 || c1 == 0xA0) ? 2 : 0;
    }
    if (s.size() >= 3) {
        const unsigned char c1 = (unsigned char)s[1], c2 = (unsigned char)s[2];
        if (c0 == 0xE1) return (c1 == 0x9A && c2 == 0x80) ? 3 : 0;
        if (c0 == 0xE2) {
            if (c1 == 0x80) return ((c2 >= 0x80 && c2 <= 0x8A) || c2 == 0xA8 || c2 == 0xA9 || c2 == 0xAF) ? 3 : 0;
            return (c1 == 0x81 && c2 == 0x9F) ? 3 : 0;
        }
        if (c0 == 0xE3) return (c1 == 0x80 && c2 == 0x80) ? 3 : 0;
    }
    return 0;
}
static size_t ws_back(std::string_view s) {
    const size_t n = s.size();
    if (!n) return 0;
    for (size_t k = 1; k <= 3 && k <= n; ++k) {
        const unsigned char lead = (unsigned char)s[n - k];
        if ((lead & 0xC0) == 0x80) continue;  // continuation byte: keep walking back
        return ws_front(s.substr(n - k)) == k ? k : 0;
    }
    return 0;
}
std::string_view rust_trim(std::string_view s) {
    for (size_t w; (w = ws_back(s)) != 0;) s.remove_suffix(w);
    for (size_t w; (w = ws_front(s)) != 0;) s.remove_prefix(w);
    return s;
}

// core::str::from_utf8 acceptance
bool is_valid_utf8(const uint8_t* p, size_t n) {
    size_t i = 0;
    while (i < n) {
        const uint8_t c = p[i];
        if (c < 0x80) { ++i; continue; }
        size_t need;
        uint32_t cp;
        if (c >= 0xC2 && c <= 0xDF) { need = 1; cp = c & 0x1F; }
        else if (c >= 0xE0 && c <= 0xEF) { need = 2; cp = c & 0x0F; }
        else if (c >= 0xF0 && c <= 0xF4) { need = 3; cp = c & 0x07; }
        else return false;
        if (i + need >= n) return false;  // truncated sequence
        for (size_t k = 1; k <= need; ++k) {
            const uint8_t d = p[i + k];
            if ((d & 0xC0) != 0x80) return false;
            cp = (cp << 6) | (d & 0x3F);
        }
        if (need == 2 && (cp < 0x800 || (cp >= 0xD800 && cp <= 0xDFFF))) return false;
        if (need == 3 && (cp < 0x10000 || cp > 0x10FFFF)) return false;
        i += need + 1;
    }
    return true;
}

static void push_utf8(std::string& s, uint32_t cp) {
    if (cp < 0x80) s.push_back((char)cp);
    else if (cp < 0x800) {
        s.push_back((char)(0xC0 | (cp >> 6)));
        s.push_back((char)(0x80 | (cp & 0x3F)));
    } else if (cp < 0x10000) {
        s.push_back((char)(0xE0 | (cp >> 12)));
        s.push_back((char)(0x80 | ((cp >> 6) & 0x3F)));
        s.push_back((char)(0x80 | (cp & 0x3F)));
    } else {
        s.push_back((char)(0xF0 | (cp >> 18)));
        s.push_back((char)(0x80 | ((cp >> 12) & 0x3F)));
        s.push_back((char)(0x80 | ((cp >> 6) & 0x3F)));
        s.push_back((char)(0x80 | (cp & 0x3F)));
    }
}
static uint32_t hex4(std::string_view v, size_t i) {
    uint32_t n = 0;
    for (size_t k = 0; k < 4; ++k) {
        const unsigned char c = (unsigned char)v[i + k];
        n = n * 16 + (c <= '9' ? c - '0' : (c | 0x20) - 'a' + 10);
    }
    return n;
}
// JSON string body (already validated by the kernel) -> String.  `nl_retry`: the line went through
// gelf_decoder.rs:44-46, where a raw LF is read as the escape `\n` and `\`+LF as `\\` followed by 'n'.
static std::string json_unescape(std::string_view v, bool nl_retry) {
    std::string res;
    res.reserve(v.size());
    for (size_t i = 0; i < v.size();) {
        const char c = v[i];
        if (c != '\\') {
            res.push_back(c);
            ++i;
            continue;
        }
        const char e = v[i + 1];
        i += 2;
        switch (e) {
            case '"': res.push_back('"'); break;
            case '\\': res.push_back('\\'); break;
            case '/': res.push_back('/'); break;
            case 'b': res.push_back('\x08'); break;
            case 'f': res.push_back('\x0c'); break;
            case 'n': res.push_back('\n'); break;
            case 'r': res.push_back('\r'); break;
            case 't': res.push_back('\t'); break;
            case 'u': {
                uint32_t n1 = hex4(v, i);
                i += 4;
                if (n1 >= 0xD800 && n1 <= 0xDBFF) {
                    const uint32_t n2 = hex4(v, i + 2);
                    i += 6;
                    n1 = (((n1 - 0xD800) << 10) | (n2 - 0xDC00)) + 0x10000;
                }
                push_utf8(res, n1);
                break;
            }
            case '\n':
                if (nl_retry) {
                    res.push_back('\\');
                    res.push_back('n');
                }
                break;
            default: break;
        }
    }
    return res;
}

// ---------------------------------------------------------------------------
// CudaBatchDecoder
// ---------------------------------------------------------------------------
CudaBatchDecoder::CudaBatchDecoder(fg_format fmt, const LtsvConfig& ltsv, const DeviceOptions& opt)
    : fmt_(fmt), ltsv_(ltsv), opt_(opt) {
    if (opt_.max_batch_bytes <= 0) opt_.max_batch_bytes = (int64_t)256 << 20;  // the C ABI's defaults (fg_create)
    if (opt_.max_batch_lines <= 0) opt_.max_batch_lines = 2 << 20;
    fg_config cfg;
    memset(&cfg, 0, sizeof cfg);
    cfg.device = opt.device;
    cfg.max_batch_bytes = opt.max_batch_bytes;
    cfg.max_batch_lines = opt.max_batch_lines;
    cfg.chunk_lines = opt.chunk_lines;
    cfg.rfc3164_year = opt.rfc3164_year;
    cfg.tzdir = opt.tzdir.empty() ? nullptr : opt.tzdir.c_str();
    cfg.input_format = (int32_t)fmt;
    std::vector<const char*> names;
    std::vector<int32_t> types;
    for (const auto& kv : ltsv.schema) {
        const int t = ltsv_type_of(kv.second);
        if (t < 0) throw std::invalid_argument("Unsupported type in input.ltsv_schema for name [" + kv.first + "]");  // ltsv_decoder.rs:44
        names.push_back(kv.first.c_str());
        types.push_back(t);
    }
    for (const auto& kv : ltsv.suffixes) {
        const int t = ltsv_type_of(kv.first);
        if (t == FG_LTSV_STRING) throw std::invalid_argument("Strings cannot be suffixed");  // :69
        if (t < 0) throw std::invalid_argument("Unsupported type in input.ltsv_suffixes for type [" + kv.first + "]");  // :74
        suffix_[t] = kv.second;
        has_suffix_[t] = true;
    }
    cfg.ltsv_has_schema = ltsv.has_schema || !ltsv.schema.empty();
    cfg.ltsv_schema_len = (int32_t)names.size();
    cfg.ltsv_schema_names = names.data();
    cfg.ltsv_schema_types = types.data();
    for (int t = 0; t < 5; ++t) cfg.ltsv_suffix[t] = has_suffix_[t] ? suffix_[t].c_str() : nullptr;
    const int rc = fg_create(&cfg, &ctx_);
    if (rc != FG_OK) {
        // No CPU fallback exists: without the CUDA library + a GPU the decoder cannot be constructed.
        throw std::runtime_error(rc == FG_E_NO_DEVICE ? "flowgger_cuda: no CUDA device (the GPU decoder has no CPU fallback)"
                                                      : "flowgger_cuda: fg_create failed");
    }
}
CudaBatchDecoder::~CudaBatchDecoder() { fg_destroy(ctx_); }

std::unique_ptr<CudaBatchDecoder> CudaBatchDecoder::make_sized(int64_t max_batch_bytes, int32_t max_batch_lines) const {
    DeviceOptions o = opt_;
    o.max_batch_bytes = max_batch_bytes;
    o.max_batch_lines = max_batch_lines;
    o.chunk_lines = 0;
    return std::unique_ptr<CudaBatchDecoder>(new CudaBatchDecoder(fmt_, ltsv_, o));
}

void CudaBatchDecoder::decode_batch(const uint8_t* bytes, const int32_t* offsets, int32_t n, fg_batch_out* out) {
    const int rc = fg_decode_batch(ctx_, fmt_, bytes, offsets, n, out);
    if (rc != FG_OK) throw std::runtime_error(std::string("fg_decode_batch: ") + fg_last_error(ctx_));
}

namespace {
// the C-ABI calls of each CudaFusedEncoder::Output, in its order
struct FusedCalls {
    const char* set_extra_name;
    int (*set_extra)(fg_ctx*, int32_t, const char* const*, const char* const*);
    const char* decode_encode_name;
    int (*decode_encode)(fg_ctx*, fg_format, const uint8_t*, const int32_t*, int32_t, fg_encoded_out*);
    const char* split_name;
    int (*split)(fg_ctx*, fg_format, fg_framing, const uint8_t*, int64_t, fg_encoded_out*, const int32_t**);
};
const FusedCalls kFusedCalls[] = {
    {"fg_set_gelf_extra: ", fg_set_gelf_extra, "fg_decode_encode_gelf: ", fg_decode_encode_gelf, "fg_split_decode_encode_gelf: ",
     fg_split_decode_encode_gelf},
    {"fg_set_ltsv_extra: ", fg_set_ltsv_extra, "fg_decode_encode_ltsv: ", fg_decode_encode_ltsv, "fg_split_decode_encode_ltsv: ",
     fg_split_decode_encode_ltsv},
    {"fg_set_capnp_extra: ", fg_set_capnp_extra, "fg_decode_encode_capnp: ", fg_decode_encode_capnp, "fg_split_decode_encode_capnp: ",
     fg_split_decode_encode_capnp},
    {"fg_set_passthrough_prefix: ", nullptr, "fg_decode_encode_passthrough: ", fg_decode_encode_passthrough,
     "fg_split_decode_encode_passthrough: ", fg_split_decode_encode_passthrough},
};
const FusedCalls& fused_calls(const CudaFusedEncoder& enc) { return kFusedCalls[(int)enc.output()]; }
}  // namespace

void CudaBatchDecoder::set_encoder(const CudaFusedEncoder& enc) {
    // set on every call: a host-side setting, and other callers of the same context may have changed it
    if (fg_set_output_framing(ctx_, enc.out_framing()) != FG_OK)
        throw std::runtime_error(std::string("fg_set_output_framing: ") + fg_last_error(ctx_));
    const FusedCalls& f = fused_calls(enc);
    if (enc.output() == CudaFusedEncoder::Output::Passthrough) {  // the header of this call, set on every call
        const std::string h = enc.header() ? enc.header()() : std::string();
        if (fg_set_passthrough_prefix(ctx_, (const uint8_t*)h.data(), (int64_t)h.size()) != FG_OK)
            throw std::runtime_error(std::string(f.set_extra_name) + fg_last_error(ctx_));
        return;
    }
    const std::vector<std::pair<std::string, std::string>>& extra = enc.extra();
    const int o = (int)enc.output();
    if (extra_valid_[o] && extra == extra_set_[o]) return;
    std::vector<const char*> k, v;
    for (const auto& kv : extra) {
        k.push_back(kv.first.c_str());
        v.push_back(kv.second.c_str());
    }
    if (f.set_extra(ctx_, (int32_t)extra.size(), k.data(), v.data()) != FG_OK)
        throw std::runtime_error(std::string(f.set_extra_name) + fg_last_error(ctx_));
    extra_set_[o] = extra;
    extra_valid_[o] = true;
}

void CudaBatchDecoder::decode_encode_gelf(const uint8_t* bytes, const int32_t* offsets, int32_t n,
                                          const std::vector<std::pair<std::string, std::string>>& extra, fg_encoded_out* out,
                                          fg_out_framing out_framing) {
    decode_encode(CudaGelfEncoder(extra, out_framing), bytes, offsets, n, out);
}

void CudaBatchDecoder::decode_encode(const CudaFusedEncoder& enc, const uint8_t* bytes, const int32_t* offsets, int32_t n,
                                     fg_encoded_out* out) {
    set_encoder(enc);
    const FusedCalls& f = fused_calls(enc);
    if (f.decode_encode(ctx_, fmt_, bytes, offsets, n, out) != FG_OK)
        throw std::runtime_error(std::string(f.decode_encode_name) + fg_last_error(ctx_));
}

const int32_t* CudaBatchDecoder::encoded_ltsv_stops() const {
    const int32_t* stop = nullptr;
    return fmt_ == FG_FMT_LTSV && fg_encoded_ltsv_stops(ctx_, &stop) == FG_OK ? stop : nullptr;
}

bool CudaBatchDecoder::try_split_decode_encode_gelf(const uint8_t* stream, int64_t nbytes, fg_framing framing,
                                                    const std::vector<std::pair<std::string, std::string>>& extra,
                                                    fg_encoded_out* out, const int32_t** line_offsets, fg_out_framing out_framing) {
    return try_split_decode_encode(CudaGelfEncoder(extra, out_framing), stream, nbytes, framing, out, line_offsets);
}

bool CudaBatchDecoder::try_split_decode_encode(const CudaFusedEncoder& enc, const uint8_t* stream, int64_t nbytes, fg_framing framing,
                                               fg_encoded_out* out, const int32_t** line_offsets) {
    set_encoder(enc);
    const FusedCalls& f = fused_calls(enc);
    const int rc = f.split(ctx_, fmt_, framing, stream, nbytes, out, line_offsets);
    if (rc == FG_E_CAPACITY) return false;
    if (rc != FG_OK) throw std::runtime_error(std::string(f.split_name) + fg_last_error(ctx_));
    return true;
}

static std::string_view span_sv(const uint8_t* bytes, fg_span s) {
    return std::string_view((const char*)bytes + s.off, (size_t)s.len);
}

DecodeResult CudaBatchDecoder::materialize(const fg_batch_out& out, const uint8_t* bytes, const int32_t* offsets,
                                           int32_t i, std::vector<std::string>* side_effects) const {
    return materialize_line(out, bytes, offsets[i], offsets[i + 1], i, side_effects);
}

void CudaBatchDecoder::split_decode(const uint8_t* stream, int64_t nbytes, fg_batch_out* out, fg_framing framing) {
    if (!try_split_decode(stream, nbytes, out, framing))
        throw std::runtime_error(std::string("fg_split_decode: ") + fg_last_error(ctx_));
}

bool CudaBatchDecoder::try_split_decode(const uint8_t* stream, int64_t nbytes, fg_batch_out* out, fg_framing framing) {
    const int rc = fg_split_decode_framed(ctx_, fmt_, framing, stream, nbytes, out);
    if (rc == FG_E_CAPACITY) return false;
    if (rc != FG_OK) throw std::runtime_error(std::string("fg_split_decode: ") + fg_last_error(ctx_));
    return true;
}

// extent of record i of a split-mode result without its terminator: "\n" / "\r\n" (BufRead::lines) or NUL
// (BufRead::split(0)); line_offsets as fg_batch_out.line_offsets
static void split_extent(const int32_t* line_offsets, const uint8_t* stream, int32_t i, int32_t& lo, int32_t& hi, fg_framing framing) {
    lo = line_offsets[i];
    hi = line_offsets[i + 1];
    if (framing == FG_FRAME_NUL) {  // BufRead::split(0): only the NUL goes
        if (hi > lo && stream[hi - 1] == 0) --hi;
        return;
    }
    if (hi > lo && stream[hi - 1] == '\n') {
        --hi;
        if (hi > lo && stream[hi - 1] == '\r') --hi;
    }
}

uint32_t row_meta(const fg_batch_out& out, int32_t i) { return out.rows5424 ? out.rows5424[i].meta : out.meta[i]; }

// Structured data of one line from 17-byte side-table rows [first, first + count) (LTSV / GELF, RFC5424 wide lines)
static void sd_from_table(fg_format fmt, const std::string* suffix, const fg_batch_out& out, const uint8_t* bytes, int32_t first,
                          int32_t count, bool nl_retry, Record& rec) {
    std::vector<StructuredData> vec;
    const bool r5 = fmt == FG_FMT_RFC5424;
    if (!r5) vec.emplace_back();  // one element with sd_id None (ltsv_decoder.rs:88, gelf_decoder.rs:35)
    for (int32_t e = first; e < first + count; ++e) {
        const uint8_t em = out.entry_meta[e];
        const uint32_t tag = em & FG_EM_TAG_MASK;
        const fg_span nm = out.entry_name[e];
        if (tag == FG_TAG_SD_HEADER) {
            vec.emplace_back();
            if (nm.off >= 0) vec.back().sd_id = std::string(span_sv(bytes, nm));
            vec.back().pairs.reserve((size_t)out.entry_val[e]);
            continue;
        }
        std::string name;
        std::string_view raw = span_sv(bytes, nm);
        if (!(em & FG_EM_NO_PREFIX)) name.push_back('_');
        if (em & FG_EM_NAME_ESC) name += json_unescape(raw, nl_retry);
        else name.append(raw);
        if ((em & FG_EM_SUFFIX) && tag >= 1 && tag <= 4) name += suffix[tag];
        SDValue v;
        v.kind = (SDValue::Kind)tag;
        const uint64_t val = out.entry_val[e];
        switch (tag) {
            case FG_TAG_STRING: {
                const uint8_t* base = (em & FG_EM_ARENA) ? out.arena : bytes;  // arena: unescaped on the device
                std::string_view sv((const char*)base + (uint32_t)(val & 0xFFFFFFFFu), (size_t)(val >> 32));
                if (em & FG_EM_UNESCAPE) v.s = json_unescape(sv, nl_retry);
                else v.s = std::string(sv);
                break;
            }
            case FG_TAG_BOOL: v.b = val != 0; break;
            case FG_TAG_F64: memcpy(&v.f, &val, 8); break;
            case FG_TAG_I64: v.i = (int64_t)val; break;
            case FG_TAG_U64: v.u = val; break;
            default: break;
        }
        vec.back().pairs.emplace_back(std::move(name), std::move(v));
    }
    rec.sd = std::move(vec);
}

// RFC5424: compact 32-byte row + 8-byte entries (include/flowgger_cuda.h: fg_row5424); wide rows carry absolute spans
static DecodeResult materialize_5424(const fg_batch_out& out, const uint8_t* bytes, int32_t line_lo, int32_t i) {
    DecodeResult r;
    const fg_row5424& row = out.rows5424[i];
    const uint32_t meta = row.meta;
    const uint32_t status = FG_META_STATUS(meta);
    if (status) {
        r.err = fg_error_string(FG_FMT_RFC5424, status);
        return r;
    }
    Record& rec = r.record;
    rec.facility = (uint8_t)FG_META_FACILITY(meta);
    rec.severity = (uint8_t)FG_META_SEVERITY(meta);
    if (FG_META_FLAGS(meta) & FG_FLAG_WIDE) {
        const fg_wide_row& w = out.wide_rows[row.sd_first];
        rec.ts = w.ts;
        rec.hostname = std::string(span_sv(bytes, w.hostname));
        rec.appname = std::string(span_sv(bytes, w.appname));
        rec.procid = std::string(span_sv(bytes, w.procid));
        rec.msgid = std::string(span_sv(bytes, w.msgid));
        if (w.msg.off >= 0) rec.msg = std::string(span_sv(bytes, w.msg));
        if (w.full_msg.off >= 0) rec.full_msg = std::string(span_sv(bytes, w.full_msg));
        if (w.sd.len > 0) sd_from_table(FG_FMT_RFC5424, nullptr, out, bytes, w.sd.off, w.sd.len, false, rec);
        return r;
    }
    rec.ts = row.ts;
    rec.hostname = std::string(span_sv(bytes, fg_row5424_field(&row, line_lo, 0)));
    rec.appname = std::string(span_sv(bytes, fg_row5424_field(&row, line_lo, 1)));
    rec.procid = std::string(span_sv(bytes, fg_row5424_field(&row, line_lo, 2)));
    rec.msgid = std::string(span_sv(bytes, fg_row5424_field(&row, line_lo, 3)));
    if (row.msg_len) rec.msg = std::string(span_sv(bytes, fg_row5424_msg(&row, line_lo)));
    rec.full_msg = std::string(span_sv(bytes, fg_row5424_full(&row, line_lo)));
    if (row.sd_count) {
        std::vector<StructuredData> vec;
        const uint8_t* line = bytes + line_lo;
        for (uint32_t e = row.sd_first; e < row.sd_first + row.sd_count; ++e) {
            const uint64_t v = out.entries8[e];
            if (v & FG_E8_HEADER) {
                vec.emplace_back();
                vec.back().sd_id = std::string((const char*)line + FG_E8_A(v), FG_E8_B(v) - FG_E8_A(v));
                vec.back().pairs.reserve(FG_E8_C(v));
                continue;
            }
            std::string name(1, '_');  // rfc5424_decoder.rs:221
            name.append((const char*)line + FG_E8_A(v), FG_E8_B(v) - FG_E8_A(v));
            SDValue val;
            val.kind = SDValue::String;
            if (v & FG_E8_ARENA) {  // value unescaped on the device (rfc5424_decoder.rs:105-125): [u16 length][bytes]
                const uint8_t* rec = out.arena + FG_E8_ARENA_OFF(v);
                uint16_t l;
                memcpy(&l, rec, 2);
                val.s.assign((const char*)rec + 2, (size_t)l);
            } else {
                val.s.assign((const char*)line + FG_E8_B(v) + 2, FG_E8_C(v) - (FG_E8_B(v) + 2));
            }
            vec.back().pairs.emplace_back(std::move(name), std::move(val));
        }
        rec.sd = std::move(vec);
    }
    return r;
}

void ltsv_missing_values(const uint8_t* bytes, int32_t lo, int32_t hi, int32_t stop, std::vector<std::string>& out) {
    for (int32_t a = lo;;) {
        int32_t b = a;
        while (b < hi && bytes[b] != '\t') ++b;
        if (a >= stop) break;
        std::string_view part((const char*)bytes + a, (size_t)(b - a));
        if (part.find(':') == std::string_view::npos) out.push_back("Missing value for name '" + std::string(part) + "'");
        if (b >= hi) break;
        a = b + 1;
    }
}

DecodeResult materialize_record(fg_format fmt, const std::string* suffix, const fg_batch_out& out, const uint8_t* bytes,
                                int32_t line_lo, int32_t line_hi, int32_t i, std::vector<std::string>* side_effects) {
    if (fmt == FG_FMT_RFC5424) return materialize_5424(out, bytes, line_lo, i);
    DecodeResult r;
    const uint32_t meta = out.meta[i];
    const uint32_t status = FG_META_STATUS(meta), flags = FG_META_FLAGS(meta);
    if (side_effects && (flags & FG_FLAG_MISSING_VALUE)) {
        // all parts when Ok / post-loop error, else the parts before the failing one
        ltsv_missing_values(bytes, line_lo, line_hi, status ? out.full_msg[i].off : line_hi + 1, *side_effects);
    }
    if (status) {
        r.err = fg_error_string(fmt, status);
        return r;
    }
    const bool nl_retry = (flags & FG_FLAG_NL_RETRY) != 0;
    Record& rec = r.record;
    rec.ts = out.ts[i];
    {
        std::string_view h = span_sv(bytes, out.hostname[i]);
        rec.hostname = (flags & FG_FLAG_HOST_ESC) ? json_unescape(h, nl_retry) : std::string(h);
    }
    if (FG_META_FACILITY(meta) != 0xFF) rec.facility = (uint8_t)FG_META_FACILITY(meta);
    if (FG_META_SEVERITY(meta) != 0xFF) rec.severity = (uint8_t)FG_META_SEVERITY(meta);
    if (out.msg[i].off >= 0) {
        if (flags & FG_FLAG_MSG_ARENA) {  // RFC3164: the tokens re-joined by single spaces on the device (rfc3164_decoder.rs:67)
            rec.msg = std::string((const char*)out.arena + out.msg[i].off, (size_t)out.msg[i].len);
        } else {
            std::string_view m = span_sv(bytes, out.msg[i]);
            rec.msg = (flags & FG_FLAG_MSG_ESC) ? json_unescape(m, nl_retry) : std::string(m);
        }
    }
    if (out.full_msg[i].off >= 0) {
        std::string_view m = span_sv(bytes, out.full_msg[i]);
        rec.full_msg = (flags & FG_FLAG_FULL_ESC) ? json_unescape(m, nl_retry) : std::string(m);
    }
    const fg_span sd = out.sd[i];
    if (sd.len > 0) sd_from_table(fmt, suffix, out, bytes, sd.off, sd.len, nl_retry, rec);
    return r;
}

DecodeResult CudaBatchDecoder::materialize_line(const fg_batch_out& out, const uint8_t* bytes, int32_t line_lo, int32_t line_hi,
                                                int32_t i, std::vector<std::string>* side_effects) const {
    return materialize_record(fmt_, suffix_, out, bytes, line_lo, line_hi, i, side_effects);
}

// GELF without "timestamp": the reference stamps the record with the wall clock (gelf_decoder.rs:109 -> utils/mod.rs:16-21)
static bool needs_wall_clock(const DecodeResult& r, const fg_batch_out& out, int32_t i) {
    return r.ok() && (FG_META_FLAGS(row_meta(out, i)) & FG_FLAG_TS_MISSING);
}
static double wall_clock_ts() {
    timespec tsn;
    clock_gettime(CLOCK_REALTIME, &tsn);
    return (double)tsn.tv_sec + (double)tsn.tv_nsec / 1e9;
}

// ---------------------------------------------------------------------------
// Decoder trait objects
// ---------------------------------------------------------------------------
CudaDecoder::CudaDecoder(fg_format fmt, const LtsvConfig& ltsv, const DeviceOptions& opt)
    : impl_(std::make_shared<CudaBatchDecoder>(fmt, ltsv, opt)) {}

DecodeResult CudaDecoder::decode(std::string_view line) const {
    const int32_t offsets[2] = {0, (int32_t)line.size()};
    fg_batch_out out;
    const uint8_t dummy = 0;
    const uint8_t* bytes = line.empty() ? &dummy : (const uint8_t*)line.data();
    // a context is single-caller and its result arrays live until the next call: clones made by clone_boxed() share it,
    // so concurrent decode() calls (one decoder clone per input thread in the reference) are serialised here
    std::lock_guard<std::mutex> guard(impl_->mutex());
    impl_->decode_batch(bytes, offsets, 1, &out);
    std::vector<std::string> fx;
    DecodeResult r = impl_->materialize(out, bytes, offsets, 0, &fx);
    for (const auto& s : fx) fprintf(stdout, "%s\n", s.c_str());
    if (needs_wall_clock(r, out, 0)) r.record.ts = wall_clock_ts();
    return r;
}
std::unique_ptr<Decoder> CudaDecoder::clone_boxed() const { return std::unique_ptr<Decoder>(new CudaDecoder(impl_)); }

// ---------------------------------------------------------------------------
// RecordEmitter, RecordBatcher + the batching splitters
// ---------------------------------------------------------------------------
namespace {

constexpr const char* kInvalidUtf8 = "Invalid UTF-8 input";  // line_splitter.rs:23, nul_splitter.rs:25

bool is_invalid_utf8_status(fg_format fmt, uint32_t status) {
    const char* s = status ? fg_error_string(fmt, status) : nullptr;
    return s && strcmp(s, kInvalidUtf8) == 0;
}

}  // namespace

RecordEmitter::RecordEmitter(const Encoder& encoder, std::function<void(std::vector<uint8_t>&&)> tx, std::ostream& err_out,
                             std::ostream& std_out, bool quiet_blank)
    : encoder_(encoder), fused_(dynamic_cast<const CudaFusedEncoder*>(&encoder)), tx_(std::move(tx)), err_(err_out),
      out_(std_out), quiet_blank_(quiet_blank) {}

const CudaFusedEncoder* RecordEmitter::fused_with(const CudaBatchDecoder& gpu) const {
    return fused_ != nullptr && CudaFusedEncoder::fuses_with(gpu.format()) ? fused_ : nullptr;
}

void RecordEmitter::emit(fg_format fmt, const fg_encoded_out& eo, const int32_t* stops, const uint8_t* bytes, int32_t i,
                         int32_t lo, int32_t hi) {
    if (stops && stops[i] >= 0) {
        fx_.clear();
        ltsv_missing_values(bytes, lo, hi, lo + stops[i], fx_);
        for (const auto& s : fx_) out_ << s << "\n";
    }
    if (eo.status[i] != 0) reject(fmt, eo.status[i], fg_error_string(fmt, eo.status[i]), bytes, lo, hi);
    else if (fused_->out_framing() == FG_OUT_NONE) tx_(std::vector<uint8_t>(eo.bytes + eo.offsets[i], eo.bytes + eo.offsets[i + 1]));
}

void RecordEmitter::end_batch(const fg_encoded_out& eo) {
    if (fused_->out_framing() != FG_OUT_NONE && eo.offsets[eo.n] > 0) tx_(std::vector<uint8_t>(eo.bytes, eo.bytes + eo.offsets[eo.n]));
}

void RecordEmitter::emit(const CudaBatchDecoder& gpu, const fg_batch_out& out, const uint8_t* bytes, int32_t i, int32_t lo,
                         int32_t hi) {
    const fg_format fmt = gpu.format();
    const uint32_t status = FG_META_STATUS(row_meta(out, i));
    if (is_invalid_utf8_status(fmt, status)) {  // never decoded, so no side effects either
        invalid_utf8();
        return;
    }
    fx_.clear();
    DecodeResult r = gpu.materialize_line(out, bytes, lo, hi, i, &fx_);
    for (const auto& s : fx_) out_ << s << "\n";
    const char* e = r.err;
    if (!e) {
        if (needs_wall_clock(r, out, i)) r.record.ts = wall_clock_ts();
        std::vector<uint8_t> enc;
        if (encoder_.encode(std::move(r.record), enc, &e)) {
            tx_(std::move(enc));
            return;
        }
    }
    reject(fmt, status, e, bytes, lo, hi);
}

void RecordEmitter::invalid_utf8() { err_ << kInvalidUtf8 << "\n"; }

// "Invalid UTF-8 input" for a record the device found not UTF-8, else "{err}: [{line.trim()}]"
void RecordEmitter::reject(fg_format fmt, uint32_t status, const char* err, const uint8_t* bytes, int32_t lo, int32_t hi) {
    if (is_invalid_utf8_status(fmt, status)) {
        invalid_utf8();
        return;
    }
    const std::string_view t = rust_trim(std::string_view((const char*)bytes + lo, (size_t)(hi - lo)));
    if (quiet_blank_ && t.empty()) return;  // nul_splitter.rs:41-45
    err_ << err << ": [" << t << "]\n";      // line_splitter.rs:37-39, nul_splitter.rs:43, syslen_splitter.rs:37
}

RecordBatcher::RecordBatcher(const Decoder& decoder, const Encoder& encoder, std::function<void(std::vector<uint8_t>&&)> tx,
                             std::ostream& err_out, std::ostream& std_out, Limits lim, bool quiet_blank)
    : gpu_(decoder.batch()), emit_(encoder, std::move(tx), err_out, std_out, quiet_blank) {
    // a batch never exceeds what the context can take (ADVICE r1: Limits used to be independent of DeviceOptions)
    max_bytes_ = std::min<int64_t>(lim.max_bytes, gpu_->capacity_bytes());
    max_lines_ = std::min<int32_t>(lim.max_lines, gpu_->capacity_lines());
    arena_.reserve((size_t)max_bytes_);
}

void RecordBatcher::flush_on(CudaBatchDecoder* gpu) {
    const int32_t n = (int32_t)offsets_.size() - 1;
    auto invalid = [&](int32_t i) {
        for (int32_t k = 0; k < invalid_before_[(size_t)i]; ++k) emit_.invalid_utf8();
    };
    if (n == 0) {
        invalid(0);
        invalid_before_.assign(1, 0);
        return;
    }
    const uint8_t dummy = 0;
    const uint8_t* bytes = arena_.empty() ? &dummy : arena_.data();
    std::lock_guard<std::mutex> guard(gpu->mutex());  // held until every Record of the batch has been materialised
    if (const CudaFusedEncoder* fused = emit_.fused_with(*gpu)) {
        // decode + encode on the device (line_splitter.rs:50-52 fused): only the encoded records come back
        fg_encoded_out eo;
        gpu->decode_encode(*fused, bytes, offsets_.data(), n, &eo);
        const int32_t* stops = gpu->encoded_ltsv_stops();
        for (int32_t i = 0; i < n; ++i) {
            invalid(i);
            emit_.emit(gpu->format(), eo, stops, bytes, i, offsets_[(size_t)i], offsets_[(size_t)i + 1]);
        }
        emit_.end_batch(eo);
    } else {
        fg_batch_out out;
        gpu->decode_batch(bytes, offsets_.data(), n, &out);
        for (int32_t i = 0; i < n; ++i) {
            invalid(i);
            emit_.emit(*gpu, out, bytes, i, offsets_[(size_t)i], offsets_[(size_t)i + 1]);
        }
    }
    invalid(n);
    arena_.clear();
    offsets_.assign(1, 0);
    invalid_before_.assign(1, 0);
}

void RecordBatcher::push(std::string_view line) {
    if ((int64_t)line.size() > max_bytes_) {
        // One record larger than a whole batch: the reference's splitters take records of any length, and there is no CPU
        // decoder to fall back on, so the record gets a context of its own, sized for it (rare, slow, correct).
        flush();
        std::unique_ptr<CudaBatchDecoder> big = gpu_->make_sized((int64_t)line.size() + 4096, 64);
        arena_.insert(arena_.end(), line.begin(), line.end());
        offsets_.push_back((int32_t)arena_.size());
        invalid_before_.push_back(0);
        flush_on(big.get());
        return;
    }
    if ((int64_t)(arena_.size() + line.size()) > max_bytes_ || (int32_t)offsets_.size() - 1 >= max_lines_) flush();
    arena_.insert(arena_.end(), line.begin(), line.end());
    offsets_.push_back((int32_t)arena_.size());
    invalid_before_.push_back(0);
}

namespace {

// The line and NUL splitters: raw blocks of the stream, each cut after its last delimiter, are framed, checked for UTF-8
// and decoded on the device (fg_split_decode_framed), with a CudaGelfEncoder on a decoder it fuses with also encoded there
// (fg_split_decode_encode_gelf).  Records, stderr and stdout come out in stream order, exactly as the reference's
// splitter + decoder + encoder give them.
class BlockSplitter {
   public:
    BlockSplitter(fg_framing framing, bool quiet_blank, const Decoder& decoder, const Encoder& encoder,
                  const std::function<void(std::vector<uint8_t>&&)>& tx, std::ostream& err_out, std::ostream& std_out)
        : framing_(framing), delim_(framing == FG_FRAME_NUL ? 0 : '\n'), gpu_(decoder.batch()),
          emit_(encoder, tx, err_out, std_out, quiet_blank) {}

    // blocks of up to `block_bytes` (at most the context's max_batch_bytes); a record longer than that grows its block
    void run(std::istream& in, int64_t block_bytes) {
        block_bytes = std::max<int64_t>(1, std::min(block_bytes, gpu_->capacity_bytes()));
        std::vector<uint8_t> buf((size_t)block_bytes);
        size_t have = 0;  // bytes in buf: the tail of the last block, then what was read since
        for (bool eof = false; !eof;) {
            if (have == buf.size()) buf.resize(buf.size() * 2);  // no delimiter in a whole buffer: a record longer than a block
            const size_t want = buf.size() - have;
            in.read((char*)buf.data() + have, (std::streamsize)want);
            const size_t got = (size_t)in.gcount();
            have += got;
            eof = got < want;
            size_t cut = have;  // at the end of the stream an unterminated last record is still a record
            if (!eof) {
                const auto last = std::find(buf.rbegin() + (std::ptrdiff_t)(buf.size() - have), buf.rend(), delim_);
                if (last == buf.rend()) continue;
                cut = (size_t)(buf.rend() - last);
            }
            if (cut) decode(gpu_.get(), buf.data(), (int64_t)cut);
            memmove(buf.data(), buf.data() + cut, have - cut);
            have -= cut;
            if (buf.size() > (size_t)block_bytes && have < (size_t)block_bytes) buf.resize((size_t)block_bytes);
        }
    }

   private:
    // records [p, p + n) in order: on `gpu` when they fit, else in two halves cut at a delimiter near the middle; a lone
    // record longer than the context gets a context of its own, sized for it (rare, slow, correct), as RecordBatcher::push
    void decode(CudaBatchDecoder* gpu, const uint8_t* p, int64_t n) {
        if (n <= gpu->capacity_bytes() && decode_on(gpu, p, n)) return;
        if (const int64_t cut = cut_near_middle(p, n)) {
            decode(gpu, p, cut);
            decode(gpu, p + cut, n - cut);
            return;
        }
        std::unique_ptr<CudaBatchDecoder> big = gpu->make_sized(n + 4096, 64);
        if (!decode_on(big.get(), p, n)) throw std::runtime_error("a record does not fit a context sized for it");
    }

    // the end of a record near the middle of [p, p + n), 0 when the block is one record (its last byte ends the last record)
    int64_t cut_near_middle(const uint8_t* p, int64_t n) const {
        const uint8_t *mid = p + n / 2, *end = p + n - 1;
        const uint8_t* f = std::find(mid, end, delim_);
        if (f != end) return f - p + 1;
        for (const uint8_t* b = mid; b > p;)
            if (*--b == delim_) return b - p + 1;
        return 0;
    }

    // false: more records than the context holds, nothing was emitted
    bool decode_on(CudaBatchDecoder* gpu, const uint8_t* p, int64_t n) {
        std::lock_guard<std::mutex> guard(gpu->mutex());  // held until every record of the block has been emitted
        int32_t lo, hi;
        if (const CudaFusedEncoder* fused = emit_.fused_with(*gpu)) {
            // framing + decode + encode on the device (line_splitter.rs:17-52 fused): only the encoded records come back
            fg_encoded_out eo;
            const int32_t* lines;
            if (!gpu->try_split_decode_encode(*fused, p, n, framing_, &eo, &lines)) return false;
            const int32_t* stops = gpu->encoded_ltsv_stops();
            for (int32_t i = 0; i < eo.n; ++i) {
                split_extent(lines, p, i, lo, hi, framing_);
                emit_.emit(gpu->format(), eo, stops, p, i, lo, hi);
            }
            emit_.end_batch(eo);
            return true;
        }
        fg_batch_out out;
        if (!gpu->try_split_decode(p, n, &out, framing_)) return false;
        for (int32_t i = 0; i < out.n; ++i) {
            split_extent(out.line_offsets, p, i, lo, hi, framing_);
            emit_.emit(*gpu, out, p, i, lo, hi);
        }
        return true;
    }

    fg_framing framing_;
    uint8_t delim_;
    std::shared_ptr<CudaBatchDecoder> gpu_;
    RecordEmitter emit_;
};

}  // namespace

void BatchingLineSplitter::run(std::istream& in, const std::function<void(std::vector<uint8_t>&&)>& tx,
                               const Decoder& decoder, const Encoder& encoder, std::ostream& err_out,
                               std::ostream& std_out) const {
    BlockSplitter(FG_FRAME_LINE, false, decoder, encoder, tx, err_out, std_out).run(in, lim_.max_bytes);
}

// splitter/nul_splitter.rs:18-47: records end at a NUL byte; the message for a rejected record is suppressed when the record is blank
void BatchingNulSplitter::run(std::istream& in, const std::function<void(std::vector<uint8_t>&&)>& tx, const Decoder& decoder,
                              const Encoder& encoder, std::ostream& err_out, std::ostream& std_out) const {
    BlockSplitter(FG_FRAME_NUL, true, decoder, encoder, tx, err_out, std_out).run(in, lim_.max_bytes);
}

// splitter/syslen_splitter.rs:17-57: octet-counted framing "<len> <record>"; the chain of lengths is sequential by nature, so
// the host walks it and the records of a batch are decoded together
void BatchingSyslenSplitter::run(std::istream& in, const std::function<void(std::vector<uint8_t>&&)>& tx, const Decoder& decoder,
                                 const Encoder& encoder, std::ostream& err_out, std::ostream& std_out) const {
    RecordBatcher batch(decoder, encoder, tx, err_out, std_out, RecordBatcher::Limits{lim_.max_lines, lim_.max_bytes});
    std::string rec;
    for (;;) {
        // read_msglen :42-57: bytes up to and including the first ' '; fewer than two => "Connection closed"
        std::string num;
        int ch;
        size_t got = 0;
        while ((ch = in.get()) != std::char_traits<char>::eof()) {
            ++got;
            if (ch == ' ') break;
            num.push_back((char)ch);
        }
        bool ok = got >= 2 && ch == ' ';
        if (got >= 2 && ch != ' ') ok = true, num.pop_back();  // read_until at EOF: the last byte plays the delimiter's role (:49)
        uint64_t len = 0;
        if (ok) {
            // usize::from_str: [+]digit+
            size_t k = 0;
            if (k < num.size() && num[k] == '+') ++k;
            ok = k < num.size();
            for (; ok && k < num.size(); ++k) {
                if (num[k] < '0' || num[k] > '9' || len > (UINT64_MAX - 9) / 10) ok = false;
                else len = len * 10 + (uint64_t)(num[k] - '0');
            }
        }
        if (!ok) {
            batch.flush();
            err_out << "Can't read message's length\n";  // :23
            return;
        }
        rec.resize((size_t)len);
        in.read(rec.data(), (std::streamsize)len);
        if ((uint64_t)in.gcount() != len) {
            batch.flush();
            err_out << "failed to fill whole buffer\n";  // read_exact's io::Error text (:27-30)
            return;
        }
        if (!is_valid_utf8((const uint8_t*)rec.data(), rec.size())) {
            // the reference unwraps String::from_utf8 here and panics (:32); the batching twin stops the stream the same way
            batch.flush();
            err_out << "Invalid UTF-8 input\n";
            return;
        }
        batch.push(rec);
    }
}

// ---------------------------------------------------------------------------
// multi-GPU sharding (SURVEY.md §8(e)): host-side split / gather only
// ---------------------------------------------------------------------------
void shard_by_bytes(const int32_t* offsets, int32_t n, int G, int32_t* bounds) {
    if (G < 1) G = 1;
    bounds[0] = 0;
    const int64_t b0 = n > 0 ? offsets[0] : 0, total = n > 0 ? (int64_t)offsets[n] - b0 : 0;
    for (int g = 1; g < G; ++g) {
        const int64_t target = b0 + total * g / G;
        // first line whose start offset is >= target
        const int32_t* it = std::lower_bound(offsets, offsets + n, (int32_t)target);
        int32_t k = (int32_t)(it - offsets);
        if (k < bounds[g - 1]) k = bounds[g - 1];
        if (k > n) k = n;
        bounds[g] = k;
    }
    bounds[G] = n;
}

MultiGpuBatchDecoder::MultiGpuBatchDecoder(fg_format fmt, const std::vector<int>& devices, const LtsvConfig& ltsv,
                                           const DeviceOptions& per_device) {
    for (int d : devices) {
        DeviceOptions o = per_device;
        o.device = d;
        dec_.emplace_back(new CudaBatchDecoder(fmt, ltsv, o));
    }
    shards_.resize(dec_.size());
}

const std::vector<MultiGpuBatchDecoder::Shard>& MultiGpuBatchDecoder::decode_batch(const uint8_t* bytes,
                                                                                  const int32_t* offsets, int32_t n) {
    const int G = (int)dec_.size();
    std::vector<int32_t> bounds((size_t)G + 1);
    shard_by_bytes(offsets, n, G, bounds.data());
    std::vector<std::thread> th;
    std::vector<std::string> errs((size_t)G);
    for (int g = 0; g < G; ++g) {
        Shard& s = shards_[(size_t)g];
        s.line0 = bounds[(size_t)g];
        s.n = bounds[(size_t)g + 1] - s.line0;
        s.byte_base = s.n > 0 ? offsets[s.line0] : 0;
        s.offsets.resize((size_t)s.n + 1);
        for (int32_t k = 0; k <= s.n; ++k) s.offsets[(size_t)k] = (int32_t)(offsets[s.line0 + k] - s.byte_base);
        if (s.n == 0) s.offsets[0] = 0;
        th.emplace_back([&, g] {
            Shard& sh = shards_[(size_t)g];
            try {
                const uint8_t dummy = 0;
                dec_[(size_t)g]->decode_batch(sh.n ? bytes + sh.byte_base : &dummy, sh.offsets.data(), sh.n, &sh.out);
            } catch (const std::exception& e) {
                errs[(size_t)g] = e.what();
            }
        });
    }
    for (auto& t : th) t.join();
    for (const auto& e : errs)
        if (!e.empty()) throw std::runtime_error(e);
    return shards_;
}

DecodeResult MultiGpuBatchDecoder::materialize(int32_t line, const uint8_t* bytes, std::vector<std::string>* fx) const {
    for (size_t g = 0; g < shards_.size(); ++g) {
        const Shard& s = shards_[g];
        if (line >= s.line0 && line < s.line0 + s.n)
            return dec_[g]->materialize(s.out, bytes + s.byte_base, s.offsets.data(), line - s.line0, fx);
    }
    DecodeResult r;
    r.err = "line out of range";
    return r;
}

// ---------------------------------------------------------------------------
// canonical dump (format documented in oracle/oracle.cpp: both sides implement it independently)
// ---------------------------------------------------------------------------
static void put_s(std::string& o, std::string_view s) {
    char b[24];
    o.append(b, (size_t)snprintf(b, sizeof b, "%zu:", s.size()));
    o.append(s);
}
static void put_o(std::string& o, const std::optional<std::string>& s) {
    if (s) put_s(o, *s);
    else o.push_back('~');
}
static void put_hex(std::string& o, double f) {
    uint64_t bits;
    memcpy(&bits, &f, 8);
    char b[24];
    o.append(b, (size_t)snprintf(b, sizeof b, "%016" PRIx64, bits));
}

void dump_result(const DecodeResult& r, bool ts_is_now, const std::vector<std::string>& fx, std::string& o) {
    char b[48];
    if (r.err) {
        o.append("E:");
        o.append(r.err);
    } else {
        const Record& rec = r.record;
        o.append("R:ts=");
        if (ts_is_now) o.append("now");
        else put_hex(o, rec.ts);
        o.append(";fac=");
        if (rec.facility) o.append(b, (size_t)snprintf(b, sizeof b, "%u", *rec.facility)); else o.push_back('~');
        o.append(";sev=");
        if (rec.severity) o.append(b, (size_t)snprintf(b, sizeof b, "%u", *rec.severity)); else o.push_back('~');
        o.append(";host="); put_s(o, rec.hostname);
        o.append(";app="); put_o(o, rec.appname);
        o.append(";proc="); put_o(o, rec.procid);
        o.append(";msgid="); put_o(o, rec.msgid);
        o.append(";msg="); put_o(o, rec.msg);
        o.append(";full="); put_o(o, rec.full_msg);
        o.append(";sd=");
        if (!rec.sd) o.push_back('~');
        else {
            o.append(b, (size_t)snprintf(b, sizeof b, "%zu", rec.sd->size()));
            for (const auto& sd : *rec.sd) {
                o.append("[id="); put_o(o, sd.sd_id);
                o.append(b, (size_t)snprintf(b, sizeof b, ";n=%zu", sd.pairs.size()));
                for (const auto& kv : sd.pairs) {
                    o.append(";k="); put_s(o, kv.first);
                    o.append(";v=");
                    const SDValue& v = kv.second;
                    switch (v.kind) {
                        case SDValue::String: o.push_back('s'); put_s(o, v.s); break;
                        case SDValue::Bool: o.append(v.b ? "b1" : "b0"); break;
                        case SDValue::F64: o.push_back('f'); put_hex(o, v.f); break;
                        case SDValue::I64: o.append(b, (size_t)snprintf(b, sizeof b, "i%" PRId64, v.i)); break;
                        case SDValue::U64: o.append(b, (size_t)snprintf(b, sizeof b, "u%" PRIu64, v.u)); break;
                        case SDValue::Null: o.push_back('n'); break;
                    }
                }
                o.push_back(']');
            }
        }
    }
    o.append(b, (size_t)snprintf(b, sizeof b, ";out=%zu", fx.size()));
    for (const auto& s : fx) { o.push_back(';'); put_s(o, s); }
}

}  // namespace flowgger

// ---------------------------------------------------------------------------
// C entry points for the Python tests / bench (ctypes)
// ---------------------------------------------------------------------------
using namespace flowgger;

namespace {

// The canonical dumps of consecutive records: their text and each one's length
struct Dumps {
    std::string text;
    std::vector<int64_t> lens;
    void add(const DecodeResult& r, bool now, const std::vector<std::string>& side_effects) {
        const size_t before = text.size();
        dump_result(r, now, side_effects, text);
        lens.push_back((int64_t)(text.size() - before));
    }
};

// `parts` concatenated in order, handed out as one malloc'd buffer and int64 offsets [records + 1] (fgh_free both)
int give_dumps(const Dumps* parts, size_t nparts, uint8_t** out_buf, int64_t** out_offsets) {
    size_t bytes = 0, n = 0;
    for (size_t t = 0; t < nparts; ++t) {
        bytes += parts[t].text.size();
        n += parts[t].lens.size();
    }
    uint8_t* buf = (uint8_t*)malloc(bytes ? bytes : 1);
    int64_t* offs = (int64_t*)malloc(sizeof(int64_t) * (n + 1));
    size_t pos = 0, li = 0;
    offs[0] = 0;
    for (size_t t = 0; t < nparts; ++t) {
        memcpy(buf + pos, parts[t].text.data(), parts[t].text.size());
        pos += parts[t].text.size();
        for (const int64_t l : parts[t].lens) {
            offs[li + 1] = offs[li] + l;
            ++li;
        }
    }
    *out_buf = buf;
    *out_offsets = offs;
    return 0;
}

}  // namespace

extern "C" {

void* fgh_decoder_new(int fmt, int device, int64_t max_bytes, int32_t max_lines, int32_t chunk_lines, int has_schema,
                      int n_schema, const char* const* names, const char* const* types, int n_suffix,
                      const char* const* suffix_types, const char* const* suffix_vals, char* errbuf, int errlen) {
    try {
        LtsvConfig lc;
        lc.has_schema = has_schema != 0;
        for (int k = 0; k < n_schema; ++k) lc.schema.emplace_back(names[k], types[k]);
        for (int k = 0; k < n_suffix; ++k) lc.suffixes.emplace_back(suffix_types[k], suffix_vals[k]);
        DeviceOptions opt;
        opt.device = device;
        opt.max_batch_bytes = max_bytes;
        opt.max_batch_lines = max_lines;
        opt.chunk_lines = chunk_lines;
        return new CudaBatchDecoder((fg_format)fmt, lc, opt);
    } catch (const std::exception& e) {
        if (errbuf && errlen > 0) snprintf(errbuf, (size_t)errlen, "%s", e.what());
        return nullptr;
    }
}
void fgh_decoder_free(void* d) { delete (CudaBatchDecoder*)d; }
fg_ctx* fgh_decoder_ctx(void* d) { return ((CudaBatchDecoder*)d)->ctx(); }
void fgh_free(void* p) { free(p); }

// materialise + canonical dump of lines [lo, hi) of a decoded batch (multi-threaded over line shards); offsets of the
// dumps are relative to the first dumped line
int fgh_dump_range(void* d, const fg_batch_out* out, const uint8_t* bytes, const int32_t* offsets, int64_t lo_line, int64_t hi_line,
                   int nthreads, uint8_t** out_buf, int64_t** out_offsets) {
    auto* dec = (CudaBatchDecoder*)d;
    const int64_t n = hi_line - lo_line;
    if (nthreads < 1) nthreads = 1;
    std::vector<Dumps> parts((size_t)nthreads);
    std::vector<std::thread> th;
    for (int t = 0; t < nthreads; ++t) {
        th.emplace_back([&, t] {
            const int64_t lo = lo_line + n * t / nthreads, hi = lo_line + n * (t + 1) / nthreads;
            Dumps& part = parts[(size_t)t];
            part.lens.reserve((size_t)(hi - lo));
            std::vector<std::string> fx;
            for (int64_t i = lo; i < hi; ++i) {
                fx.clear();
                DecodeResult r = dec->materialize(*out, bytes, offsets, (int32_t)i, &fx);
                part.add(r, needs_wall_clock(r, *out, (int32_t)i), fx);
            }
        });
    }
    for (auto& x : th) x.join();
    return give_dumps(parts.data(), parts.size(), out_buf, out_offsets);
}
int fgh_dump_out(void* d, const fg_batch_out* out, const uint8_t* bytes, const int32_t* offsets, int nthreads,
                 uint8_t** out_buf, int64_t** out_offsets) {
    return fgh_dump_range(d, out, bytes, offsets, 0, out->n, nthreads, out_buf, out_offsets);
}

// same dump from bare result arrays (no context, no device): lets the CPU test-suite run the product's materialiser
// over rows produced by the device-logic emulation (tests/emu)
int fgh_dump_records(int fmt, const fg_batch_out* out, const uint8_t* bytes, const int32_t* offsets, const char* const* ltsv_suffix,
                     uint8_t** out_buf, int64_t** out_offsets) {
    std::string suffix[5];  // input.ltsv_suffixes by fg_ltsv_type (nullptr: none)
    for (int t = 1; t < 5 && ltsv_suffix; ++t)
        if (ltsv_suffix[t]) suffix[t] = ltsv_suffix[t];
    Dumps dumps;
    std::vector<std::string> fx;
    for (int32_t i = 0; i < out->n; ++i) {
        fx.clear();
        DecodeResult r = materialize_record((fg_format)fmt, suffix, *out, bytes, offsets[i], offsets[i + 1], i, &fx);
        dumps.add(r, needs_wall_clock(r, *out, i), fx);
    }
    return give_dumps(&dumps, 1, out_buf, out_offsets);
}

// materialisation rate (owned Records, like the reference builds them), for the e2e report
double fgh_materialize_bench(void* d, const fg_batch_out* out, const uint8_t* bytes, const int32_t* offsets,
                             int nthreads) {
    auto* dec = (CudaBatchDecoder*)d;
    const int64_t n = out->n;
    if (nthreads < 1) nthreads = 1;
    std::vector<std::thread> th;
    std::vector<uint64_t> sink((size_t)nthreads, 0);
    timespec t0, t1;
    clock_gettime(CLOCK_MONOTONIC, &t0);
    for (int t = 0; t < nthreads; ++t) {
        th.emplace_back([&, t] {
            const int64_t lo = n * t / nthreads, hi = n * (t + 1) / nthreads;
            uint64_t s = 0;
            for (int64_t i = lo; i < hi; ++i) {
                DecodeResult r = dec->materialize(*out, bytes, offsets, (int32_t)i, nullptr);
                s += r.record.hostname.size();
            }
            sink[(size_t)t] = s;
        });
    }
    for (auto& x : th) x.join();
    clock_gettime(CLOCK_MONOTONIC, &t1);
    return (double)(t1.tv_sec - t0.tv_sec) + (double)(t1.tv_nsec - t0.tv_nsec) * 1e-9;
}

// fg_split_decode + canonical dumps of every line (split-mode twin of fgh_dump_out); also returns the line offsets
int fgh_split_dump(void* d, int framing, const uint8_t* stream, int64_t nbytes, uint8_t** out_buf, int64_t** out_offsets, int32_t** out_line_offsets,
                   int32_t* out_n, float* kernel_ms, char* errbuf, int errlen) {
    auto* dec = (CudaBatchDecoder*)d;
    try {
        fg_batch_out out;
        dec->split_decode(stream, nbytes, &out, (fg_framing)framing);
        const int32_t n = out.n;
        Dumps dumps;
        std::vector<std::string> fx;
        for (int32_t i = 0; i < n; ++i) {
            int32_t lo, hi;
            split_extent(out.line_offsets, stream, i, lo, hi, (fg_framing)framing);
            fx.clear();
            DecodeResult r = dec->materialize_line(out, stream, lo, hi, i, &fx);
            dumps.add(r, needs_wall_clock(r, out, i), fx);
        }
        int32_t* lo_out = (int32_t*)malloc(sizeof(int32_t) * ((size_t)n + 1));
        memcpy(lo_out, out.line_offsets, sizeof(int32_t) * ((size_t)n + 1));
        give_dumps(&dumps, 1, out_buf, out_offsets);
        *out_line_offsets = lo_out;
        *out_n = n;
        if (kernel_ms) *kernel_ms = out.kernel_ms;
        return 0;
    } catch (const std::exception& e) {
        if (errbuf && errlen > 0) snprintf(errbuf, (size_t)errlen, "%s", e.what());
        return -1;
    }
}

// Decoder::clone_boxed() drop-in check: `nthreads` clones of one CudaDecoder, each decoding its interleaved share of the
// lines through Decoder::decode (a batch of one per call), as the reference's per-connection threads do; canonical dumps
// come back in line order
int fgh_clone_decode_threads(int fmt, int device, const uint8_t* bytes, const int32_t* offsets, int32_t n, int nthreads,
                             uint8_t** out_buf, int64_t** out_offsets, char* errbuf, int errlen) {
    try {
        DeviceOptions opt;
        opt.device = device;
        opt.max_batch_bytes = 1 << 20;
        opt.max_batch_lines = 1024;
        CudaDecoder root((fg_format)fmt, {}, opt);
        std::vector<std::unique_ptr<Decoder>> clones;
        for (int t = 0; t < nthreads; ++t) clones.push_back(root.clone_boxed());
        std::vector<DecodeResult> results((size_t)n);
        std::vector<std::thread> th;
        std::vector<std::string> errs((size_t)nthreads);
        for (int t = 0; t < nthreads; ++t) {
            th.emplace_back([&, t] {
                try {
                    for (int32_t i = t; i < n; i += nthreads) {
                        std::string_view line((const char*)bytes + offsets[i], (size_t)(offsets[i + 1] - offsets[i]));
                        results[(size_t)i] = clones[(size_t)t]->decode(line);
                    }
                } catch (const std::exception& e) {
                    errs[(size_t)t] = e.what();
                }
            });
        }
        for (auto& x : th) x.join();
        for (const auto& e : errs)
            if (!e.empty()) throw std::runtime_error(e);
        Dumps dumps;
        for (const DecodeResult& r : results) dumps.add(r, false, {});
        return give_dumps(&dumps, 1, out_buf, out_offsets);
    } catch (const std::exception& e) {
        if (errbuf && errlen > 0) snprintf(errbuf, (size_t)errlen, "%s", e.what());
        return -1;
    }
}

}  // extern "C"

namespace {

// The harness of the splitter entries: BatchingLineSplitter (framing 0), BatchingNulSplitter (framing 1) or
// BatchingSyslenSplitter (framing 2, through RecordBatcher) over `text` with `enc`; `tx` receives what the splitter sends
int run_splitter(void* d, const uint8_t* text, int64_t len, int32_t max_lines, int64_t max_bytes, int framing, const Encoder& enc,
                 const std::function<void(std::vector<uint8_t>&&)>& tx, std::string& err, std::string& out) {
    struct Shared : Decoder {
        std::shared_ptr<CudaBatchDecoder> b;
        DecodeResult decode(std::string_view) const override { return {}; }
        std::unique_ptr<Decoder> clone_boxed() const override { return nullptr; }
        std::shared_ptr<CudaBatchDecoder> batch() const override { return b; }
    } dec;
    dec.b = std::shared_ptr<CudaBatchDecoder>((CudaBatchDecoder*)d, [](CudaBatchDecoder*) {});
    BatchingLineSplitter::Limits lim;
    lim.max_lines = max_lines;
    lim.max_bytes = max_bytes;
    std::string in((const char*)text, (size_t)len);
    std::istringstream is(in);
    std::ostringstream es, os;
    try {
        if (framing == 1) BatchingNulSplitter(lim).run(is, tx, dec, enc, es, os);        // input.framing = "nul"
        else if (framing == 2) BatchingSyslenSplitter(lim).run(is, tx, dec, enc, es, os);  // input.framing = "syslen"
        else BatchingLineSplitter(lim).run(is, tx, dec, enc, es, os);                      // input.framing = "line"
    } catch (const std::exception&) {
        return -1;
    }
    err = es.str();
    out = os.str();
    return 0;
}

std::vector<std::pair<std::string, std::string>> extra_of(int n_extra, const char* const* keys, const char* const* vals) {
    std::vector<std::pair<std::string, std::string>> extra;
    for (int k = 0; k < n_extra; ++k) extra.emplace_back(keys[k], vals[k]);
    return extra;
}

void give(const std::string& s, uint8_t** p, int64_t* n) {
    *p = (uint8_t*)malloc(s.size() ? s.size() : 1);
    memcpy(*p, s.data(), s.size());
    *n = (int64_t)s.size();
}

}  // namespace

extern "C" {

// BatchingLineSplitter (framing 0), BatchingNulSplitter (framing 1) or BatchingSyslenSplitter (framing 2, through
// RecordBatcher) with output.format = "gelf" (fused decode + encode): text in, one JSON record per line, stderr and
// stdout text out
int fgh_splitter_run_gelf(void* d, const uint8_t* text, int64_t len, int32_t max_lines, int64_t max_bytes, int n_extra,
                          const char* const* keys, const char* const* vals, uint8_t** out_records, int64_t* out_records_len,
                          uint8_t** out_stderr, int64_t* out_stderr_len, int framing, uint8_t** out_stdout, int64_t* out_stdout_len) {
    std::string records, err, out;
    auto tx = [&](std::vector<uint8_t>&& v) { records.append(v.begin(), v.end()); records.push_back('\n'); };
    if (run_splitter(d, text, len, max_lines, max_bytes, framing, CudaGelfEncoder(extra_of(n_extra, keys, vals)), tx, err, out))
        return -1;
    give(records, out_records, out_records_len);
    give(err, out_stderr, out_stderr_len);
    give(out, out_stdout, out_stdout_len);
    return 0;
}

// fgh_splitter_run_gelf with output.framing (fg_out_framing) applied on the device: the output stream exactly as the
// splitter sent it (no separator added), stderr and stdout text
int fgh_splitter_run_gelf_framed(void* d, const uint8_t* text, int64_t len, int32_t max_lines, int64_t max_bytes, int n_extra,
                                 const char* const* keys, const char* const* vals, int framing, int out_framing, uint8_t** out_stream,
                                 int64_t* out_stream_len, uint8_t** out_stderr, int64_t* out_stderr_len, uint8_t** out_stdout,
                                 int64_t* out_stdout_len) {
    std::string stream, err, out;
    auto tx = [&](std::vector<uint8_t>&& v) { stream.append(v.begin(), v.end()); };
    const CudaGelfEncoder enc(extra_of(n_extra, keys, vals), (fg_out_framing)out_framing);
    if (run_splitter(d, text, len, max_lines, max_bytes, framing, enc, tx, err, out)) return -1;
    give(stream, out_stream, out_stream_len);
    give(err, out_stderr, out_stderr_len);
    give(out, out_stdout, out_stdout_len);
    return 0;
}

// fgh_splitter_run_gelf_framed with output.format = "ltsv" (CudaLtsvEncoder): the output stream exactly as the splitter
// sent it, stderr and stdout text
int fgh_splitter_run_ltsv_framed(void* d, const uint8_t* text, int64_t len, int32_t max_lines, int64_t max_bytes, int n_extra,
                                 const char* const* keys, const char* const* vals, int framing, int out_framing, uint8_t** out_stream,
                                 int64_t* out_stream_len, uint8_t** out_stderr, int64_t* out_stderr_len, uint8_t** out_stdout,
                                 int64_t* out_stdout_len) {
    std::string stream, err, out;
    auto tx = [&](std::vector<uint8_t>&& v) { stream.append(v.begin(), v.end()); };
    const CudaLtsvEncoder enc(extra_of(n_extra, keys, vals), (fg_out_framing)out_framing);
    if (run_splitter(d, text, len, max_lines, max_bytes, framing, enc, tx, err, out)) return -1;
    give(stream, out_stream, out_stream_len);
    give(err, out_stderr, out_stderr_len);
    give(out, out_stdout, out_stdout_len);
    return 0;
}

// fgh_splitter_run_gelf_framed with output.format = "capnp" (CudaCapnpEncoder)
int fgh_splitter_run_capnp_framed(void* d, const uint8_t* text, int64_t len, int32_t max_lines, int64_t max_bytes, int n_extra,
                                  const char* const* keys, const char* const* vals, int framing, int out_framing, uint8_t** out_stream,
                                  int64_t* out_stream_len, uint8_t** out_stderr, int64_t* out_stderr_len, uint8_t** out_stdout,
                                  int64_t* out_stdout_len) {
    std::string stream, err, out;
    auto tx = [&](std::vector<uint8_t>&& v) { stream.append(v.begin(), v.end()); };
    const CudaCapnpEncoder enc(extra_of(n_extra, keys, vals), (fg_out_framing)out_framing);
    if (run_splitter(d, text, len, max_lines, max_bytes, framing, enc, tx, err, out)) return -1;
    give(stream, out_stream, out_stream_len);
    give(err, out_stderr, out_stderr_len);
    give(out, out_stdout, out_stdout_len);
    return 0;
}

// fgh_splitter_run_gelf_framed with output.format = "passthrough" (CudaPassthroughEncoder): `header` [header_len] is
// the header of every device call, none when NULL
int fgh_splitter_run_passthrough_framed(void* d, const uint8_t* text, int64_t len, int32_t max_lines, int64_t max_bytes,
                                        const uint8_t* header, int64_t header_len, int framing, int out_framing, uint8_t** out_stream,
                                        int64_t* out_stream_len, uint8_t** out_stderr, int64_t* out_stderr_len, uint8_t** out_stdout,
                                        int64_t* out_stdout_len) {
    std::string stream, err, out;
    auto tx = [&](std::vector<uint8_t>&& v) { stream.append(v.begin(), v.end()); };
    std::function<std::string()> source;
    if (header) source = [h = std::string((const char*)header, (size_t)header_len)] { return h; };
    const CudaPassthroughEncoder enc(std::move(source), (fg_out_framing)out_framing);
    if (run_splitter(d, text, len, max_lines, max_bytes, framing, enc, tx, err, out)) return -1;
    give(stream, out_stream, out_stream_len);
    give(err, out_stderr, out_stderr_len);
    give(out, out_stdout, out_stdout_len);
    return 0;
}

int fgh_is_valid_utf8(const uint8_t* p, int64_t n) { return is_valid_utf8(p, (size_t)n) ? 1 : 0; }

void fgh_shard_by_bytes(const int32_t* offsets, int32_t n, int G, int32_t* bounds) { shard_by_bytes(offsets, n, G, bounds); }

// multi-GPU fan-out: decode on `ndev` devices and return the canonical dumps in batch order
int fgh_multi_decode_dump(int fmt, const int* devices, int ndev, int64_t max_bytes, int32_t max_lines,
                          const uint8_t* bytes, const int32_t* offsets, int32_t n, uint8_t** out_buf,
                          int64_t** out_offsets, char* errbuf, int errlen) {
    try {
        DeviceOptions opt;
        opt.max_batch_bytes = max_bytes;
        opt.max_batch_lines = max_lines;
        MultiGpuBatchDecoder dec((fg_format)fmt, std::vector<int>(devices, devices + ndev), {}, opt);
        const auto& shards = dec.decode_batch(bytes, offsets, n);
        Dumps dumps;
        std::vector<std::string> fx;
        size_t g = 0;
        for (int32_t i = 0; i < n; ++i) {
            fx.clear();
            DecodeResult r = dec.materialize(i, bytes, &fx);
            while (g + 1 < shards.size() && i >= shards[g].line0 + shards[g].n) ++g;  // the shard that holds line i
            dumps.add(r, needs_wall_clock(r, shards[g].out, i - shards[g].line0), fx);
        }
        return give_dumps(&dumps, 1, out_buf, out_offsets);
    } catch (const std::exception& e) {
        if (errbuf && errlen > 0) snprintf(errbuf, (size_t)errlen, "%s", e.what());
        return -1;
    }
}

// BatchingLineSplitter twin of LineSplitter::run for tests: text in, one canonical dump line per record out
// (encoder = the parity dump), stderr/stdout text of the reference captured.
int fgh_splitter_run(void* d, int framing, const uint8_t* text, int64_t len, int32_t max_lines, int64_t max_bytes, uint8_t** out_records,
                     int64_t* out_records_len, uint8_t** out_stderr, int64_t* out_stderr_len, uint8_t** out_stdout,
                     int64_t* out_stdout_len) {
    struct DumpEncoder : Encoder {
        bool encode(Record&& rec, std::vector<uint8_t>& out, const char**) const override {
            DecodeResult r;
            r.record = std::move(rec);
            std::string s;
            dump_result(r, false, {}, s);
            out.assign(s.begin(), s.end());
            return true;
        }
    };
    std::string records, err, out;
    auto tx = [&](std::vector<uint8_t>&& v) { records.append(v.begin(), v.end()); records.push_back('\n'); };
    if (run_splitter(d, text, len, max_lines, max_bytes, framing, DumpEncoder(), tx, err, out)) return -1;
    give(records, out_records, out_records_len);
    give(err, out_stderr, out_stderr_len);
    give(out, out_stdout, out_stdout_len);
    return 0;
}

}  // extern "C"
