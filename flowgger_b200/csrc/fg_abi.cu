// fg_abi.cu — the C ABI declared in include/flowgger_cuda.h.
//
// Host side of the drop-in boundary: owns the device buffers, pinned host
// result arrays and streams of one context, pipelines host<->device copies
// with the parse kernels chunk by chunk, and exposes the device-resident
// variant used for roofline measurement.  There is no CPU parsing anywhere in
// this file: if CUDA is unavailable every entry point returns an error.
#include <cuda_runtime.h>

#include <algorithm>
#include <chrono>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <ctime>
#include <mutex>
#include <new>
#include <string>
#include <utility>
#include <vector>

#include "../../include/flowgger_cuda.h"
#include "fg_capnp_layout.cuh"
#include "fg_kernels.cuh"
#include "fg_status.h"
#include "fg_rfc3164.cuh"
#include "fg_tz.h"

namespace {

// The reference's `&'static str` for every status (file:line in flowgger src/flowgger/decoder/)
const char* kErrorStrings[FG_ST_COUNT] = {};
struct ErrorTableInit {
    ErrorTableInit() {
        auto& t = kErrorStrings;
        t[FG_E5_BOM] = "Unsupported BOM";                                        // rfc5424_decoder.rs:69
        t[FG_E5_PRI_BRACKETS] = "The priority should be inside brackets";         // :76
        t[FG_E5_INVALID_PRI] = "Invalid priority";                                // :83
        t[FG_E5_MISSING_VERSION] = "Missing version";                             // :84
        t[FG_E5_UNSUPPORTED_VERSION] = "Unsupported version";                     // :86
        t[FG_E5_MISSING_TS] = "Missing timestamp";                                // :25
        t[FG_E5_BAD_TS] = "Unable to parse the date from RFC3339 to Unix time in RFC5424 decoder";  // :97
        t[FG_E5_MISSING_HOST] = "Missing hostname";                               // :26
        t[FG_E5_MISSING_APP] = "Missing application name";                        // :27
        t[FG_E5_MISSING_PROCID] = "Missing process id";                           // :28
        t[FG_E5_MISSING_MSGID] = "Missing message id";                            // :29
        t[FG_E5_MISSING_DATA] = "Missing message data";                           // :30
        t[FG_E5_MISSING_MSG] = "Missing log message";                             // :129,:148
        t[FG_E5_MALFORMED] = "Malformated RFC5424 message";                       // :154,:159
        t[FG_E5_MISSING_SD] = "Missing structured data";                          // :177
        t[FG_E5_SD_FORMAT] = "Format error in the structured data";               // :235
        t[FG_E5_SD_NO_END] = "Missing ] after structured data";                   // :239
        t[FG_E5_MISSING_PRI_VERSION] = "Missing priority and version";            // :24 (unreachable)
        t[FG_E5_EMPTY_PRI] = "Empty priority";                                    // :81 (unreachable)
        t[FG_E5_MISSING_SD_ID] = "Missing structured data id";                    // :176 (unreachable)
        t[FG_EL_TS] = "Unable to parse the English to Unix timestamp in LTSV decoder";  // ltsv_decoder.rs:252
        t[FG_EL_SEV] = "Invalid severity level";                                  // :116
        t[FG_EL_SEV_HIGH] = "Severity level should be <= 7";                      // :118
        t[FG_EL_BOOL] = "Type error; boolean was expected";                       // :143
        t[FG_EL_F64] = "Type error; f64 was expected";                            // :159
        t[FG_EL_I64] = "Type error; i64 was expected";                            // :175
        t[FG_EL_U64] = "Type error; u64 was expected";                            // :191
        t[FG_EL_MISSING_TS] = "Missing timestamp";                                // :205
        t[FG_EL_MISSING_HOST] = "Missing hostname";                               // :206
        t[FG_EG_JSON] = "Invalid GELF input, unable to parse as a JSON object";   // gelf_decoder.rs:49
        t[FG_EG_EMPTY] = "Empty GELF input";                                      // :50
        t[FG_EG_TS] = "Invalid GELF timestamp";                                   // :53
        t[FG_EG_HOST] = "GELF host name must be a string";                        // :58
        t[FG_EG_SHORT] = "GELF short message must be a string";                   // :66
        t[FG_EG_FULL] = "GELF full message must be a string";                     // :74
        t[FG_EG_VERSION_T] = "GELF version must be a string";                     // :78
        t[FG_EG_VERSION] = "Unsupported GELF version";                            // :80
        t[FG_EG_SEV] = "Invalid severity level";                                  // :83
        t[FG_EG_SEV_HIGH] = "Invalid severity level (too high)";                  // :85
        t[FG_EG_SD_TYPE] = "Invalid value type in structured data";               // :97
        t[FG_EG_MISSING_HOST] = "Missing hostname";                               // :110
        t[FG_ES_INVALID_UTF8] = "Invalid UTF-8 input";                            // splitter/line_splitter.rs:23
        t[FG_E3_PRI_MALFORMED] = "Malformed RFC3164 event: Invalid priority";     // rfc3164_decoder.rs:131
        t[FG_E3_PRI_INVALID] = "Invalid priority";                                // :137
        t[FG_E3_CUSTOM] = "Malformed RFC3164 event: Invalid timestamp or hostname";  // :120
        t[FG_E3_TIME_FORMAT] = "Invalid time format";                             // :158
        t[FG_E3_WITH_YEAR] = "Unable to parse RFC3164 date with year";            // :178
        t[FG_E3_DATE] = "Unable to parse the date in RFC3164 decoder";            // :211
        t[FG_E3_PANIC] = "(the reference panics here: index out of bounds, rfc3164_decoder.rs:64)";
    }
} g_error_table_init;

constexpr size_t kPad = 256;            // slack after the device byte buffer (16-byte bulk-copy granules)
constexpr size_t kBounceBytes = 32u << 20;  // pinned bounce buffers for pageable caller memory
constexpr size_t kL2FlushBytes = 256u << 20;
constexpr size_t kCountBytes = sizeof(uint32_t) * fg::K5_COUNT;  // one snapshot of the counter block

enum Where { DEV = 1, HOST = 2, BOTH = 3 };

// A device array, a pinned host array, or both of the same length (the host one mirrors the device one); freed when
// it is dropped or reallocated.
template <class T, class H = T>
struct Buf {
    static_assert(sizeof(T) == sizeof(H), "the pinned mirror has the layout of the device array");
    T* d = nullptr;
    H* h = nullptr;
    size_t n = 0;  // elements, once allocated
    Buf() = default;
    Buf(const Buf&) = delete;
    Buf& operator=(const Buf&) = delete;
    ~Buf() { reset(); }
    void reset() {
        if (d) cudaFree(d);
        if (h) cudaFreeHost(h);
        d = nullptr;
        h = nullptr;
        n = 0;
    }
    cudaError_t alloc(size_t count, Where w) {
        reset();
        cudaError_t e = (w & DEV) ? cudaMalloc((void**)&d, count * sizeof(T)) : cudaSuccess;
        if (e == cudaSuccess && (w & HOST)) e = cudaHostAlloc((void**)&h, count * sizeof(H), cudaHostAllocDefault);
        if (e == cudaSuccess) n = count;
        return e;
    }
};

void destroy(cudaEvent_t e) { cudaEventDestroy(e); }
void destroy(cudaStream_t s) { cudaStreamDestroy(s); }
// An owned event or stream
template <class H>
struct Handle {
    H h = nullptr;
    Handle() = default;
    Handle(Handle&& o) noexcept : h(o.h) { o.h = nullptr; }
    Handle(const Handle&) = delete;
    Handle& operator=(const Handle&) = delete;
    ~Handle() {
        if (h) destroy(h);
    }
    operator H() const { return h; }
};
using Event = Handle<cudaEvent_t>;
using Stream = Handle<cudaStream_t>;

// the events of one parse step of a pipelined call
struct StepEvents {
    Event h2d;     // its input is on the device
    Event k0, k1;  // bracket its kernels
    Event cnt;     // its counter snapshot is on the host
};

// Side tables: the kernels bump-allocate their rows through a word of the counter block, which keeps counting past the
// capacity when a batch does not fit; the batch is then redone after a regrow to the reported need.  A table is up to
// three columns (device array + pinned mirror) of `width` bytes per row that share one capacity.
enum { T_ENTRIES, T_E8, T_ARENA, T_WIDE, T_COUNT };
struct TableShape {
    size_t width[3];
    size_t round;  // rows are allocated in multiples of this
};
constexpr TableShape kTableShape[T_COUNT] = {
    {{sizeof(fg_span), sizeof(uint64_t), 1}, 256},  // T_ENTRIES: 17-byte rows (LTSV, GELF, RFC5424 wide lines)
    {{sizeof(uint64_t), 0, 0}, 256},                // T_E8: RFC5424 8-byte entries
    {{1, 0, 0}, 256},                               // T_ARENA: RFC5424 unescaped values, RFC3164 re-joined messages
    {{sizeof(fg_wide_row), 0, 0}, 1},               // T_WIDE: RFC5424 wide rows
};
static_assert(sizeof(fg_span) == sizeof(int2) && sizeof(fg_wide_row) == sizeof(fg::WideRow), "pinned rows mirror the device rows");
struct Table {
    Buf<uint8_t> col[3];
    size_t cap = 0;  // rows
};

// The tables a format uses, the counter that fills each (-1: none, the table stays empty) and its size on first use,
// max(max_bytes / div, floor) rows (`grow`: also whenever it is smaller than that)
struct TableUse {
    int table, counter;
    size_t div, floor;
    bool grow;
};
struct FormatTables {
    int n;
    TableUse use[4];
    const TableUse* begin() const { return use; }
    const TableUse* end() const { return use + n; }
};
constexpr FormatTables kFormatTables[4] = {
    {4, {{T_E8, fg::K5_ENTRIES, 24, 4096, false}, {T_ARENA, fg::K5_ARENA, 64, 64 << 10, false},
         {T_WIDE, fg::K5_WIDE_ROWS, 0, 1024, false}, {T_ENTRIES, fg::K5_WIDE_ENTRIES, 0, 4096, false}}},  // RFC5424
    {1, {{T_ENTRIES, fg::K5_ENTRIES, 24, 4096, true}}},                                                  // LTSV
    {1, {{T_ENTRIES, fg::K5_ENTRIES, 24, 4096, true}}},                                                  // GELF
    {2, {{T_ARENA, fg::K5_ARENA, 32, 64 << 10, false}, {T_ENTRIES, -1, 0, 256, false}}},                 // RFC3164
};

}  // namespace

struct fg_ctx {
    int device = 0;
    size_t max_bytes = 0;
    int max_lines = 0;
    int chunk_lines = 0;
    int input_format = 0;  // fg_config.input_format
    Stream s_h2d, s_comp, s_d2h;
    Stream s_parse;  // split mode: the parse kernels, behind the framing on s_comp
    Event ev_a, ev_b;
    Event ev_dom0, ev_dom1;  // bracket the dominant kernel of a resident step
    Event ev_s0, ev_s1;      // bracket the framing of a split call
    std::vector<StepEvents> steps;
    std::vector<Event> ev_split;  // split mode: chunk k is framed and validated
    Event bounce_ev[2];
    Buf<uint8_t> bounce[2];   // pinned bounce buffers
    Buf<uint32_t> counts;     // pinned per-step snapshots of the counter block (K5_COUNT words each)
    // device: input
    Buf<uint8_t> bytes;
    Buf<int32_t> offsets;
    Buf<uint32_t> k;  // counter block (fg::K5_*)
    Buf<uint8_t> flush;
    // side tables
    Table tab[T_COUNT];
    // LTSV / GELF / RFC3164: columnar rows (9 columns sized for max_lines); LTSV / GELF: scratch side-table rows
    Buf<uint8_t> rows;
    Buf<int2> tmp_name;  // provisional side-table rows, indexed by byte offset / scratch_div
    Buf<unsigned long long> tmp_val;
    Buf<uint8_t> tmp_meta;
    // RFC5424: compact rows, work lists (the wide list is also GELF's slow list)
    Buf<fg::Row5424, fg_row5424> rows5;
    Buf<uint32_t> esc_list, wide_list;
    // fused GELF encoder (fg_decode_encode_gelf)
    Buf<unsigned long long> enc_lens, enc_rel;  // record lengths and their sum inside a launch: a launch may pass 4 GiB
    Buf<unsigned long long> enc_base;  // [chunks + 1] running output size
    Buf<uint8_t> enc_out;
    size_t enc_out_cap = 0;  // enc_out holds 16 bytes more
    Buf<long long, int64_t> enc_offsets;
    Buf<uint8_t> enc_status;
    Buf<int32_t> enc_stop;  // LTSV: where the decoder stopped printing "Missing value" lines (fg_encoded_ltsv_stops)
    int enc_stop_n = -1;    // records of the last fused LTSV call (-1: the last fused call was not LTSV)
    double gelf_now = 0.0;  // GELF: Record.ts of the call's records without "timestamp" (fg_encoded_gelf_now)
    bool gelf_now_ok = false;  // the last fused call was on GELF input and succeeded
    Buf<uint8_t> scan_temp;
    size_t scan_temp_bytes = 0;
    Buf<uint8_t> static_blob;  // fixed GELF keys + output.gelf_extra, sorted
    int n_static = 0;
    const int32_t* d_static_key_off = nullptr;
    const int32_t* d_static_lit_off = nullptr;
    const int32_t* d_static_kind = nullptr;
    std::vector<std::pair<std::string, std::string>> gelf_extra;
    Buf<uint8_t> ltsv_extra;   // output.ltsv_extra as the one literal the LTSV encoder writes (fg_set_ltsv_extra)
    int ltsv_extra_len = 0;
    // output.capnp_extra (fg_set_capnp_extra): key 0, value 0, key 1, ... and their bounds [2n + 1], sorted by key
    Buf<uint8_t> capnp_extra;
    const int32_t* d_capnp_extra_off = nullptr;
    int capnp_extra_n = 0;
    // the header of every passthrough record (fg_set_passthrough_prefix)
    Buf<uint8_t> pt_prefix;
    int32_t pt_prefix_len = 0;
    fg_out_framing out_framing = FG_OUT_NONE;  // output.framing of the fused encoder (fg_set_output_framing)
    // split mode (fg_split_decode)
    Buf<uint32_t> seg;
    Buf<int32_t> n_lines;
    Buf<uint8_t> invalid;
    Buf<int32_t> split_offsets;  // pinned: the line offsets found on the device
    Buf<int32_t> cum;
    float last_split_ms = 0.f;
    // RFC3164: the year `now_utc().year()` stands for (0: read the clock at every call) and the zone database
    int r3164_year = 0;
    int call_year = 1970;  // the year of the call in progress (current_year())
    std::string tzdir;
    fg::TzHostTable tz_host;
    Buf<uint8_t> tz_blob;
    fg::TzDeviceTable tz_dev{};
    // LTSV config blob
    Buf<uint8_t> ltsv_blob;
    fg::LtsvDeviceConfig ltsv{};
    float last_dom_ms = 0.f;
    // resident batch
    int res_n = 0;
    size_t res_bytes = 0;
    int res_fmt = -1;
    uint32_t res_tot[fg::K5_COUNT] = {};
    std::string last_error;
    int64_t launches = 0;
    int max_tile5 = 0;  // RFC5424: tile + bitmap must fit the opt-in shared memory
    int num_sms = 0;    // of the device: the post kernels' fixed grids stride over their work lists with a few CTAs per SM
};

namespace {

constexpr int kColW[9] = {8, 4, 8, 8, 8, 8, 8, 8, 8};  // ts(8) meta(4) host app proc msgid msg full sd (8 each)
enum { C_TS = 0, C_META, C_HOST, C_APP, C_PROC, C_MSGID, C_MSG, C_FULL, C_SD, C_COUNT };
size_t col_off(const fg_ctx* c, int col) {
    const size_t n = (size_t)c->max_lines;
    size_t o = 0;
    for (int k = 0; k < col; ++k) o += (size_t)kColW[k] * n;
    return o;
}

int fail(fg_ctx* c, int code, const char* what, cudaError_t e = cudaSuccess) {
    if (c) {
        c->last_error = what;
        if (e != cudaSuccess) {
            c->last_error += ": ";
            c->last_error += cudaGetErrorString(e);
        }
    }
    return code;
}

#define FG_CUDA(ctx, call)                                         \
    do {                                                           \
        cudaError_t _e = (call);                                   \
        if (_e != cudaSuccess) return fail(ctx, FG_E_CUDA, #call, _e); \
    } while (0)

cudaError_t create(Event& e, unsigned flags) { return cudaEventCreateWithFlags(&e.h, flags); }
cudaError_t create(Stream& s) { return cudaStreamCreateWithFlags(&s.h, cudaStreamNonBlocking); }

template <class T>
T* dev(const fg_ctx* c, int t, int col = 0) {
    return reinterpret_cast<T*>(c->tab[t].col[col].d);
}
template <class T>
T* host(const fg_ctx* c, int t, int col = 0) {
    return reinterpret_cast<T*>(c->tab[t].col[col].h);
}
uint32_t cap32(const fg_ctx* c, int t) { return (uint32_t)std::min<size_t>(c->tab[t].cap, 0xFFFFFFFFu); }

// (re)allocates table t for `rows` rows; its old columns are all freed first
int grow_table(fg_ctx* c, int t, size_t rows) {
    const TableShape& S = kTableShape[t];
    Table& T = c->tab[t];
    T.cap = 0;
    for (auto& col : T.col) col.reset();
    rows = (rows + S.round - 1) / S.round * S.round;
    for (int i = 0; i < 3 && S.width[i]; ++i) FG_CUDA(c, T.col[i].alloc(rows * S.width[i], BOTH));
    T.cap = rows;
    return FG_OK;
}

// tables whose fill level the kernels report in the counter block
bool tables_overflow(const fg_ctx* c, int fmt, const uint32_t* t) {
    for (const TableUse& u : kFormatTables[fmt])
        if (u.counter >= 0 && t[u.counter] > c->tab[u.table].cap) return true;
    return false;
}
int regrow_tables(fg_ctx* c, int fmt, const uint32_t* t) {
    for (const TableUse& u : kFormatTables[fmt]) {
        const size_t need = u.counter >= 0 ? t[u.counter] : 0;
        if (need > c->tab[u.table].cap)
            if (int rc = grow_table(c, u.table, need + need / 8 + 1024)) return rc;
    }
    return FG_OK;
}

// side tables: the rows a chunk produced are the contiguous range [prev, cur) of each bump allocator
int copy_tables_d2h(fg_ctx* c, int fmt, const uint32_t* prev, const uint32_t* cur, cudaStream_t s) {
    for (const TableUse& u : kFormatTables[fmt]) {
        if (u.counter < 0 || cur[u.counter] <= prev[u.counter]) continue;
        const size_t from = prev[u.counter], rows = cur[u.counter] - prev[u.counter];
        const TableShape& S = kTableShape[u.table];
        const Table& T = c->tab[u.table];
        for (int i = 0; i < 3 && S.width[i]; ++i)
            FG_CUDA(c, cudaMemcpyAsync(T.col[i].h + from * S.width[i], T.col[i].d + from * S.width[i], rows * S.width[i],
                                       cudaMemcpyDeviceToHost, s));
    }
    return FG_OK;
}

// Host arrays placed at 16-byte aligned offsets of one device blob, uploaded at once.  A zeroed 16-byte tail follows
// the last array: device code may read whole words past the end of an array.
struct Packer {
    std::vector<uint8_t> bytes;
    template <class V>
    size_t add(const V& v) {
        const size_t at = bytes.size();
        const uint8_t* src = reinterpret_cast<const uint8_t*>(v.data());
        bytes.insert(bytes.end(), src, src + v.size() * sizeof(v[0]));
        bytes.resize((bytes.size() + 15) & ~(size_t)15, 0);
        return at;
    }
    int upload(fg_ctx* c, Buf<uint8_t>& blob) {
        bytes.resize(bytes.size() + 16, 0);
        FG_CUDA(c, blob.alloc(bytes.size(), DEV));
        FG_CUDA(c, cudaMemcpy(blob.d, bytes.data(), bytes.size(), cudaMemcpyHostToDevice));
        return FG_OK;
    }
};

// packed zone table -> one device blob (fg::TzDeviceTable points into it)
int upload_tz(fg_ctx* c) {
    const fg::TzHostTable& H = c->tz_host;
    Packer p;
    const size_t o_hash = p.add(H.hash), o_key = p.add(H.key), o_zone = p.add(H.zone), o_noff = p.add(H.name_off),
                 o_first = p.add(H.first), o_off = p.add(H.off), o_names = p.add(H.names);
    if (int rc = p.upload(c, c->tz_blob)) return rc;
    const uint8_t* b = c->tz_blob.d;
    fg::TzDeviceTable& T = c->tz_dev;
    T = H.view();
    T.hash = (const unsigned long long*)(b + o_hash);
    T.key = (const long long*)(b + o_key);
    T.zone = (const int32_t*)(b + o_zone);
    T.name_off = (const int32_t*)(b + o_noff);
    T.first = (const int32_t*)(b + o_first);
    T.off = (const int32_t*)(b + o_off);
    T.names = b + o_names;
    return FG_OK;
}

// LTSV schema / suffixes -> one device blob
int upload_ltsv_config(fg_ctx* c, const fg_config* cfg) {
    std::vector<uint8_t> names, suffix;
    std::vector<int32_t> name_off{0}, types;
    const int ns = (cfg->ltsv_schema_names && cfg->ltsv_schema_types) ? cfg->ltsv_schema_len : 0;
    for (int k = 0; k < ns; ++k) {
        const char* s = cfg->ltsv_schema_names[k];
        names.insert(names.end(), (const uint8_t*)s, (const uint8_t*)s + strlen(s));
        name_off.push_back((int32_t)names.size());
        types.push_back(cfg->ltsv_schema_types[k]);
    }
    fg::LtsvDeviceConfig& L = c->ltsv;
    L.has_schema = (cfg->ltsv_has_schema || ns > 0) ? 1 : 0;
    L.n_schema = ns;
    L.suffix_present = 0;
    L.suffix_off[0] = 0;
    for (int t = 0; t < 5; ++t) {
        const char* s = cfg->ltsv_suffix[t];
        if (t > 0 && s) {
            L.suffix_present |= 1u << t;
            suffix.insert(suffix.end(), (const uint8_t*)s, (const uint8_t*)s + strlen(s));
        }
        L.suffix_off[t + 1] = (int32_t)suffix.size();
    }
    Packer p;
    const size_t o_names = p.add(names), o_off = p.add(name_off), o_types = p.add(types), o_suf = p.add(suffix);
    if (int rc = p.upload(c, c->ltsv_blob)) return rc;
    const uint8_t* b = c->ltsv_blob.d;
    L.names = b + o_names;
    L.name_off = (const int32_t*)(b + o_off);
    L.types = (const int32_t*)(b + o_types);
    L.suffix = b + o_suf;
    return FG_OK;
}

// `OffsetDateTime::now_utc().year()` (rfc3164_decoder.rs:175): the configured year, else the clock's, once per call
int current_year(const fg_ctx* c) {
    if (c->r3164_year != 0) return c->r3164_year;
    const time_t now = time(nullptr);
    struct tm g;
    gmtime_r(&now, &g);
    return g.tm_year + 1900;
}

// Format-specific buffers are allocated on first use of the format.
int ensure_format(fg_ctx* c, int fmt) {
    const size_t L = (size_t)c->max_lines;
    if (fmt == FG_FMT_RFC5424) {
        if (!c->rows5.d) {
            FG_CUDA(c, c->rows5.alloc(L, BOTH));
            FG_CUDA(c, c->esc_list.alloc(L, DEV));
            FG_CUDA(c, c->wide_list.alloc(L, DEV));
        }
    } else if (!c->rows.d) {
        FG_CUDA(c, c->rows.alloc(col_off(c, C_COUNT), BOTH));
    }
    if (fmt == FG_FMT_GELF && !c->wide_list.d) FG_CUDA(c, c->wide_list.alloc(L, DEV));  // slow list
    for (const TableUse& u : kFormatTables[fmt]) {
        const size_t first = u.div ? std::max<size_t>(c->max_bytes / u.div, u.floor) : u.floor;
        const size_t cap = c->tab[u.table].cap;
        if (u.grow ? cap < first : !cap)
            if (int rc = grow_table(c, u.table, first)) return rc;
    }
    if (fmt == FG_FMT_RFC3164) {  // zone names need the database
        if (!c->tz_host.loaded) {
            std::string err;
            if (!fg::tz_load_dir(c->tzdir.empty() ? nullptr : c->tzdir.c_str(), c->tz_host, err)) return fail(c, FG_E_ARG, err.c_str());
        }
        if (!c->tz_blob.d)
            if (int rc = upload_tz(c)) return rc;
    }
    if (fmt == FG_FMT_LTSV || fmt == FG_FMT_GELF) {
        // Scratch table for provisional side-table rows, indexed by byte offset (see Format<>::scratch_index):
        // a row needs >= 3 input bytes in GELF, >= 1 byte + its TAB in LTSV.
        const size_t need = (fmt == FG_FMT_LTSV ? c->max_bytes / 2 + L : c->max_bytes / 3) + 64;
        if (c->tmp_meta.n < need) {  // allocated last: set once all three exist
            c->tmp_name.reset(); c->tmp_val.reset(); c->tmp_meta.reset();
            FG_CUDA(c, c->tmp_name.alloc(need, DEV));
            FG_CUDA(c, c->tmp_val.alloc(need, DEV));
            FG_CUDA(c, c->tmp_meta.alloc(need, DEV));
        }
    }
    return FG_OK;
}

// validate the format, then the context's device, the format's buffers and the year of this call
int begin_call(fg_ctx* c, fg_format fmt) {
    if ((int)fmt < 0 || (int)fmt > 3) return fail(c, FG_E_ARG, "unknown format");
    FG_CUDA(c, cudaSetDevice(c->device));
    if (int rc = ensure_format(c, (int)fmt)) return rc;
    c->call_year = current_year(c);
    return FG_OK;
}

// shared-memory tile: mean span of a CTA's lines plus 2 % slack; the kernel handles whatever does not fit in extra rounds
int pick_tile(const fg_ctx* c, size_t total_bytes, int n, int fmt) {
    const double mean = n > 0 ? (double)total_bytes / n : 0.0;
    const long lines = fg::lines_per_cta(fmt), gran = 8 * lines;  // 1 KiB steps for 128-line CTAs, 512 B for 64
    const int max_tile[4] = {c->max_tile5, fg::kLtsvMaxTile, fg::kGelfMaxTile, fg::kR3164MaxTile};
    long t = (long)(mean * lines * 1.02) + gran;
    t = (t + gran - 1) / gran * gran;
    t = std::max(t, 8L * 1024);
    t = std::min(t, (long)max_tile[fmt]);
    return (int)t;
}

// One parse launch over lines [line0, line0 + n) of the resident offsets (for RFC5424: parse + unescape + wide kernels)
int launch_lines(fg_ctx* c, int fmt, int line0, int n, int tile, const uint8_t* invalid, int strip_eol, cudaStream_t s,
                 bool time_dominant = false) {
    if (fmt == FG_FMT_RFC5424) {
        fg::Parse5424Params P;
        P.bytes = c->bytes.d;
        P.offsets = c->offsets.d + line0;
        P.n = n;
        P.tile_bytes = tile;
        P.rows = reinterpret_cast<uint4*>(c->rows5.d + line0);
        P.entries = dev<unsigned long long>(c, T_E8);
        P.entry_cap = cap32(c, T_E8);
        P.counters = c->k.d;
        P.esc_list = c->esc_list.d;
        P.wide_list = c->wide_list.d;
        P.arena = dev<uint8_t>(c, T_ARENA);
        P.arena_cap = cap32(c, T_ARENA);
        P.wide_rows = dev<fg::WideRow>(c, T_WIDE);
        P.wide_cap = cap32(c, T_WIDE);
        P.wentry_name = dev<int2>(c, T_ENTRIES, 0);
        P.wentry_val = dev<unsigned long long>(c, T_ENTRIES, 1);
        P.wentry_meta = dev<uint8_t>(c, T_ENTRIES, 2);
        P.wentry_cap = cap32(c, T_ENTRIES);
        P.line0 = line0;
        P.bad_offsets = c->k.d + fg::K5_BAD_OFFSETS;
        P.line_invalid = invalid;
        P.strip_eol = strip_eol;
        P.num_sms = c->num_sms;
        FG_CUDA(c, cudaMemsetAsync(c->k.d + fg::K5_ESC_LIST, 0, 8, s));  // the two work lists are per launch
        FG_CUDA(c, fg::launch_parse5424(P, s, time_dominant ? c->ev_dom0.h : nullptr, time_dominant ? c->ev_dom1.h : nullptr));
        c->launches += 2;  // parse5424_kernel + post5424_kernel
        return FG_OK;
    }
    fg::ParseParams P;
    P.bytes = c->bytes.d;
    P.offsets = c->offsets.d + line0;
    P.n = n;
    P.line0 = line0;
    P.tile_bytes = tile;
    P.num_sms = c->num_sms;
    uint8_t* r = c->rows.d;
    P.ts = (double*)(r + col_off(c, C_TS)) + line0;
    P.meta = (uint32_t*)(r + col_off(c, C_META)) + line0;
    P.host = (int2*)(r + col_off(c, C_HOST)) + line0;
    P.app = (int2*)(r + col_off(c, C_APP)) + line0;
    P.proc = (int2*)(r + col_off(c, C_PROC)) + line0;
    P.msgid = (int2*)(r + col_off(c, C_MSGID)) + line0;
    P.msg = (int2*)(r + col_off(c, C_MSG)) + line0;
    P.full = (int2*)(r + col_off(c, C_FULL)) + line0;
    P.sd = (int2*)(r + col_off(c, C_SD)) + line0;
    P.entry_name = dev<int2>(c, T_ENTRIES, 0);
    P.entry_val = dev<unsigned long long>(c, T_ENTRIES, 1);
    P.entry_meta = dev<uint8_t>(c, T_ENTRIES, 2);
    P.tmp_name = c->tmp_name.d;
    P.tmp_val = c->tmp_val.d;
    P.tmp_meta = c->tmp_meta.d;
    P.line_invalid = invalid;
    P.strip_eol = strip_eol;
    P.entry_counter = c->k.d + fg::K5_ENTRIES;
    P.entry_cap = cap32(c, T_ENTRIES);
    P.bad_offsets = c->k.d + fg::K5_BAD_OFFSETS;
    P.slow_list = c->wide_list.d;
    P.slow_count = c->k.d + fg::K5_WIDE_LIST;
    if (fmt == FG_FMT_GELF) FG_CUDA(c, cudaMemsetAsync(c->k.d + fg::K5_WIDE_LIST, 0, 4, s));  // the work list is per launch
    P.ltsv = c->ltsv;
    P.r3164.year = c->call_year;
    P.r3164.tz = c->tz_dev;
    P.r3164.arena = dev<uint8_t>(c, T_ARENA);
    P.r3164.arena_cap = cap32(c, T_ARENA);
    P.r3164.arena_counter = c->k.d + fg::K5_ARENA;
    if (time_dominant) FG_CUDA(c, cudaEventRecord(c->ev_dom0, s));
    FG_CUDA(c, fg::launch_parse(fmt, P, s));
    if (time_dominant) FG_CUDA(c, cudaEventRecord(c->ev_dom1, s));
    c->launches += fmt == FG_FMT_GELF ? 2 : 1;  // GELF: parse_gelf_kernel + post_gelf_kernel
    return FG_OK;
}

// The decoders whose device-resident results the fused GELF encoder reads.  LTSV only on a context created for it: the
// pair keys carry that context's ltsv_suffixes.  GELF likewise, the rule LTSV follows.
int check_fusable(fg_ctx* c, int fmt) {
    if (fmt == FG_FMT_RFC5424 || fmt == FG_FMT_RFC3164 || ((fmt == FG_FMT_LTSV || fmt == FG_FMT_GELF) && c->input_format == fmt))
        return FG_OK;
    return fail(c, FG_E_ARG, "the fused encoder takes input.format = rfc5424");
}

// Start of a fused GELF call: the LTSV stops and the wall clock of an earlier call end here, whatever this one returns.
// gelf_decoder.rs:109 -> utils/mod.rs:16-21: the wall clock as secs + nanos / 1e9, read once at the start of a fused GELF
// call for all its records without "timestamp"
void begin_fused(fg_ctx* c, int fmt) {
    c->enc_stop_n = -1;
    c->gelf_now_ok = false;
    if (fmt != FG_FMT_GELF) return;
    timespec t;
    clock_gettime(CLOCK_REALTIME, &t);
    c->gelf_now = (double)t.tv_sec + (double)t.tv_nsec / 1e9;
}

// The encoder a pipelined call runs after each parse step: none (the rows and side tables come back), or the GELF, LTSV,
// Cap'n Proto or passthrough encoder (only the encoded records come back)
enum Enc { ENC_NONE = 0, ENC_GELF = 1, ENC_LTSV = 2, ENC_CAPNP = 3, ENC_PASSTHROUGH = 4 };

// the word of the counter block (past the K5_COUNT snapshotted ones) where the Cap'n Proto encoder reports the least
// offset of a line whose record capnp cannot hold (0xFFFFFFFF: none)
constexpr int kCapnpTooLong = 16;

// The fused encoder `enc` over the decoder's results of lines [l0, l0 + n), parse step k
int launch_encode(fg_ctx* c, int enc, int fmt, int k, int l0, int n, int tile, cudaStream_t s) {
    fg::GelfEncodeParams E{};
    E.bytes = c->bytes.d;
    E.offsets = c->offsets.d + l0;
    E.n = n;
    if (fmt == FG_FMT_RFC5424) {
        E.rows = reinterpret_cast<const uint4*>(c->rows5.d + l0);
    } else {
        const uint8_t* r = c->rows.d;
        E.col_ts = (const double*)(r + col_off(c, C_TS)) + l0;
        E.col_meta = (const uint32_t*)(r + col_off(c, C_META)) + l0;
        E.col_host = (const int2*)(r + col_off(c, C_HOST)) + l0;
        E.col_msg = (const int2*)(r + col_off(c, C_MSG)) + l0;
        E.col_full = (const int2*)(r + col_off(c, C_FULL)) + l0;
    }
    if (fmt == FG_FMT_LTSV || fmt == FG_FMT_GELF) E.col_sd = (const int2*)(c->rows.d + col_off(c, C_SD)) + l0;
    if (fmt == FG_FMT_GELF) {
        E.gelf_now = c->gelf_now;
        E.gelf_entries = c->k.d + fg::K5_ENTRIES;
        // a line longer than the LTSV encoder's segment length field (2^29 - 1 bytes, the GELF encoder's is 2^30 - 1) may
        // hold a string with escapes that no segment holds: long_json_span_kernel looks for one.  The passthrough
        // encoder has no segment length field.
        if ((enc == ENC_GELF || enc == ENC_LTSV) && c->max_bytes >= ((size_t)1 << 29)) E.long_json_span = c->k.d + fg::K5_LONG_JSON_SPAN;
    }
    if (fmt == FG_FMT_LTSV) {
        E.ltsv_suffix = c->ltsv.suffix;
        for (int t = 0; t < 6; ++t) E.ltsv_suffix_off[t] = c->ltsv.suffix_off[t];
        E.ltsv_stop = c->enc_stop.d + l0;
    }
    E.entries = dev<unsigned long long>(c, T_E8);
    E.arena = dev<uint8_t>(c, T_ARENA);
    E.wide_rows = dev<fg::WideRow>(c, T_WIDE);
    E.wentry_name = dev<int2>(c, T_ENTRIES, 0);
    E.wentry_val = dev<unsigned long long>(c, T_ENTRIES, 1);
    E.wentry_meta = dev<uint8_t>(c, T_ENTRIES, 2);
    if (enc == ENC_GELF) {
        E.static_blob = c->static_blob.d;
        E.n_static = c->n_static;
        E.static_key_off = c->d_static_key_off;
        E.static_lit_off = c->d_static_lit_off;
        E.static_kind = c->d_static_kind;
    } else if (enc == ENC_LTSV) {
        E.static_blob = c->ltsv_extra.d;
        E.n_static = c->ltsv_extra_len;
    } else if (enc == ENC_CAPNP) {
        E.static_blob = c->capnp_extra.d;
        E.n_static = c->capnp_extra_n;
        E.static_key_off = c->d_capnp_extra_off;
        E.long_json_span = c->k.d + kCapnpTooLong;
    } else {
        E.static_blob = c->pt_prefix.d;
        E.n_static = c->pt_prefix_len;
    }
    E.lens = c->enc_lens.d + l0;
    E.rel = c->enc_rel.d + l0;
    E.base = c->enc_base.d + k;
    E.out = c->enc_out.d;
    E.out_cap = c->enc_out_cap;
    E.out_offsets = c->enc_offsets.d + l0;
    E.status = c->enc_status.d + l0;
    E.bad_offsets = c->k.d + fg::K5_BAD_OFFSETS;
    E.entry_cap = cap32(c, T_E8);
    E.wide_cap = cap32(c, T_WIDE);
    E.wentry_cap = cap32(c, T_ENTRIES);
    E.arena_cap = cap32(c, T_ARENA);
    E.out_framing = (int32_t)c->out_framing;
    // the encoder's CTAs take 256 lines (4 x the parse kernel's 64); configure_gelf_encode allowed max_tile5
    E.tile_bytes = std::min(4 * tile, c->max_tile5);
    if (enc == ENC_GELF) FG_CUDA(c, fg::launch_gelf_encode(fmt, E, c->scan_temp.d, c->scan_temp_bytes, s));
    else if (enc == ENC_LTSV) FG_CUDA(c, fg::launch_ltsv_encode(fmt, E, c->scan_temp.d, c->scan_temp_bytes, s));
    else if (enc == ENC_CAPNP) FG_CUDA(c, fg::launch_capnp_encode(fmt, E, c->scan_temp.d, c->scan_temp_bytes, s));
    else FG_CUDA(c, fg::launch_passthrough_encode(fmt, E, c->scan_temp.d, c->scan_temp_bytes, s));
    c->launches += E.long_json_span && enc != ENC_CAPNP ? 5 : 4;
    return FG_OK;
}

bool col_used(int col) { return !(col == C_APP || col == C_PROC || col == C_MSGID); }  // LTSV / GELF have no such fields

void fill_out(fg_ctx* c, int fmt, int n, const uint32_t* tot, fg_batch_out* out) {
    out->n = n;
    for (const TableUse& u : kFormatTables[fmt]) {
        const uint32_t rows = u.counter >= 0 ? tot[u.counter] : 0;
        switch (u.table) {
            case T_ENTRIES:
                out->entry_name = host<fg_span>(c, T_ENTRIES, 0);
                out->entry_val = host<uint64_t>(c, T_ENTRIES, 1);
                out->entry_meta = host<uint8_t>(c, T_ENTRIES, 2);
                out->n_entries = (int32_t)rows;
                break;
            case T_E8:
                out->entries8 = host<uint64_t>(c, T_E8);
                out->n_entries8 = (int32_t)rows;
                break;
            case T_ARENA:
                out->arena = host<uint8_t>(c, T_ARENA);
                out->arena_bytes = (int64_t)rows;
                break;
            case T_WIDE:
                out->wide_rows = host<fg_wide_row>(c, T_WIDE);
                out->n_wide = (int32_t)rows;
                break;
        }
    }
    if (fmt == FG_FMT_RFC5424) {
        out->rows5424 = c->rows5.h;
        return;
    }
    uint8_t* r = c->rows.h;
    out->ts = (const double*)(r + col_off(c, C_TS));
    out->meta = (const uint32_t*)(r + col_off(c, C_META));
    out->hostname = (const fg_span*)(r + col_off(c, C_HOST));
    out->msg = (const fg_span*)(r + col_off(c, C_MSG));
    out->full_msg = (const fg_span*)(r + col_off(c, C_FULL));
    out->sd = (const fg_span*)(r + col_off(c, C_SD));
}

int copy_rows_d2h(fg_ctx* c, int fmt, int line0, int n, cudaStream_t s) {
    if (n <= 0) return FG_OK;
    if (fmt == FG_FMT_RFC5424) {
        FG_CUDA(c, cudaMemcpyAsync(c->rows5.h + line0, c->rows5.d + line0, (size_t)n * 32, cudaMemcpyDeviceToHost, s));
        return FG_OK;
    }
    // ts and meta: one copy each; the 8-byte span columns share one pitch (8 * max_lines), so every run of consecutive
    // used span columns goes back as ONE 2-D copy (few large D2H operations disturb the concurrent H2D stream less)
    for (int col = C_TS; col <= C_META; ++col) {
        const size_t o = col_off(c, col) + (size_t)line0 * kColW[col];
        FG_CUDA(c, cudaMemcpyAsync(c->rows.h + o, c->rows.d + o, (size_t)n * kColW[col], cudaMemcpyDeviceToHost, s));
    }
    const size_t pitch = (size_t)c->max_lines * 8;
    int col = C_HOST;
    while (col < C_COUNT) {
        if (!col_used(col)) { ++col; continue; }
        int end = col;
        while (end + 1 < C_COUNT && col_used(end + 1)) ++end;
        const size_t o = col_off(c, col) + (size_t)line0 * 8;
        FG_CUDA(c, cudaMemcpy2DAsync(c->rows.h + o, pitch, c->rows.d + o, pitch, (size_t)n * 8, (size_t)(end - col + 1),
                                     cudaMemcpyDeviceToHost, s));
        col = end + 1;
    }
    return FG_OK;
}

bool is_pinned(const void* p) {
    cudaPointerAttributes a;
    if (cudaPointerGetAttributes(&a, p) != cudaSuccess) {
        cudaGetLastError();
        return false;
    }
    return a.type == cudaMemoryTypeHost;
}

// H2D of an arbitrary host range: direct DMA when pinned, else through two pinned bounce buffers
int h2d(fg_ctx* c, void* dst, const void* src, size_t bytes, bool pinned, int& bounce_ix) {
    if (!bytes) return FG_OK;
    if (pinned) {
        FG_CUDA(c, cudaMemcpyAsync(dst, src, bytes, cudaMemcpyHostToDevice, c->s_h2d));
        return FG_OK;
    }
    size_t done = 0;
    while (done < bytes) {
        const size_t k = std::min(kBounceBytes, bytes - done);
        const int b = bounce_ix & 1;
        FG_CUDA(c, cudaEventSynchronize(c->bounce_ev[b]));
        memcpy(c->bounce[b].h, (const uint8_t*)src + done, k);
        FG_CUDA(c, cudaMemcpyAsync((uint8_t*)dst + done, c->bounce[b].h, k, cudaMemcpyHostToDevice, c->s_h2d));
        FG_CUDA(c, cudaEventRecord(c->bounce_ev[b], c->s_h2d));
        done += k;
        ++bounce_ix;
    }
    return FG_OK;
}

// events and counter snapshots for `steps` parse steps
int ensure_steps(fg_ctx* c, int steps) {
    while ((int)c->steps.size() < steps) {
        StepEvents e;
        FG_CUDA(c, create(e.h2d, cudaEventDisableTiming));
        FG_CUDA(c, create(e.k0, cudaEventDefault));
        FG_CUDA(c, create(e.k1, cudaEventDefault));
        FG_CUDA(c, create(e.cnt, cudaEventDisableTiming));
        c->steps.push_back(std::move(e));
    }
    if (c->counts.n < (size_t)steps * fg::K5_COUNT) FG_CUDA(c, c->counts.alloc((size_t)steps * fg::K5_COUNT, HOST));
    return FG_OK;
}

// Cheap host-side checks; the interior of the offsets array is checked on the device (check_offsets_kernel) next to
// the parse, so a non-monotone or out-of-range offset fails the call with FG_E_ARG instead of reaching a kernel.
int check_batch(fg_ctx* c, const uint8_t* bytes, const int32_t* offsets, int32_t n) {
    if (!c) return FG_E_ARG;
    if (n < 0 || (n > 0 && (!bytes || !offsets))) return fail(c, FG_E_ARG, "null input");
    if (n > c->max_lines) return fail(c, FG_E_CAPACITY, "batch has more lines than max_batch_lines");
    if (n > 0) {
        if (offsets[0] < 0 || offsets[n] < offsets[0]) return fail(c, FG_E_ARG, "offsets must be non-negative and non-decreasing");
        if ((size_t)offsets[n] > c->max_bytes) return fail(c, FG_E_CAPACITY, "batch has more bytes than max_batch_bytes");
    }
    return FG_OK;
}

// A caller's batch of lines, uploaded chunk by chunk
struct HostBatch {
    const uint8_t* bytes;
    const int32_t* offsets;
    bool pin_b, pin_o;
    int bounce_ix;
};

// Parse step k's input: H2D of lines [l0, l1) on s_h2d, then the device check of their offsets on s_comp
int upload_chunk(fg_ctx* c, HostBatch& B, int k, int l0, int l1) {
    const size_t b0 = (size_t)B.offsets[l0], b1 = (size_t)B.offsets[l1];
    if (b1 < b0 || b1 > c->max_bytes) {
        cudaDeviceSynchronize();
        return fail(c, FG_E_ARG, "offsets must be non-decreasing and within max_batch_bytes");
    }
    if (int rc = h2d(c, c->bytes.d + b0, B.bytes + b0, b1 - b0, B.pin_b, B.bounce_ix)) return rc;
    if (int rc = h2d(c, c->offsets.d + l0, B.offsets + l0, sizeof(int32_t) * (size_t)(l1 - l0 + 1), B.pin_o, B.bounce_ix)) return rc;
    FG_CUDA(c, cudaEventRecord(c->steps[k].h2d, c->s_h2d));
    FG_CUDA(c, cudaStreamWaitEvent(c->s_comp, c->steps[k].h2d, 0));
    FG_CUDA(c, fg::launch_check_offsets(c->offsets.d + l0, l1 - l0, (long long)c->max_bytes, c->k.d + fg::K5_BAD_OFFSETS, c->s_comp));
    return FG_OK;
}

// Parse step k of a pipelined call on stream s: the kernels over lines [l0, l0 + n) between the step's timing events
// (with `encode`, the GELF encoder after the parse), the counter snapshot, then on s_d2h once the snapshot is in: the
// rows, or the encoder's statuses and record offsets
int parse_step(fg_ctx* c, int fmt, int k, int l0, int n, int tile, const uint8_t* invalid, int strip, cudaStream_t s,
               int encode) {
    StepEvents& e = c->steps[k];
    FG_CUDA(c, cudaEventRecord(e.k0, s));
    if (int rc = launch_lines(c, fmt, l0, n, tile, invalid, strip, s)) return rc;
    if (encode)
        if (int rc = launch_encode(c, encode, fmt, k, l0, n, tile, s)) return rc;
    FG_CUDA(c, cudaEventRecord(e.k1, s));
    FG_CUDA(c, cudaMemcpyAsync(c->counts.h + (size_t)k * fg::K5_COUNT, c->k.d, kCountBytes, cudaMemcpyDeviceToHost, s));
    if (encode)
        FG_CUDA(c, cudaMemcpyAsync(c->enc_base.h + k + 1, c->enc_base.d + k + 1, sizeof(unsigned long long), cudaMemcpyDeviceToHost, s));
    FG_CUDA(c, cudaEventRecord(e.cnt, s));
    FG_CUDA(c, cudaStreamWaitEvent(c->s_d2h, e.cnt, 0));
    if (!encode) return copy_rows_d2h(c, fmt, l0, n, c->s_d2h);
    FG_CUDA(c, cudaMemcpyAsync(c->enc_status.h + l0, c->enc_status.d + l0, (size_t)n, cudaMemcpyDeviceToHost, c->s_d2h));
    FG_CUDA(c, cudaMemcpyAsync(c->enc_offsets.h + l0, c->enc_offsets.d + l0, (size_t)(n + 1) * 8, cudaMemcpyDeviceToHost, c->s_d2h));
    if (fmt == FG_FMT_LTSV)
        FG_CUDA(c, cudaMemcpyAsync(c->enc_stop.h + l0, c->enc_stop.d + l0, (size_t)n * 4, cudaMemcpyDeviceToHost, c->s_d2h));
    return FG_OK;
}

const uint32_t kZeroCounts[fg::K5_COUNT] = {};

// How far the drain of one attempt has got: the next parse step, the counters the last drained one left, whether a step
// overflowed
struct Drain {
    bool encode;
    int next = 0;
    const uint32_t* prev = kZeroCounts;
    bool overflow = false;
};

Drain begin_drain(fg_ctx* c, int encode) {
    if (encode) c->enc_base.h[0] = 0;
    return Drain{encode != ENC_NONE};
}

// Waits for the counter snapshots of the parse steps before `upto` in order and copies what each step produced back on
// s_d2h while later steps are still in flight: its range [prev, cur) of every side table, or with `encode` its encoded
// records, the range [base(k), base(k+1)) of the output.  After an overflow nothing more is copied, but every snapshot
// is still waited for.
int drain_upto(fg_ctx* c, int fmt, int upto, Drain& d) {
    for (; d.next < upto; ++d.next) {
        const int k = d.next;
        FG_CUDA(c, cudaEventSynchronize(c->steps[k].cnt));
        const uint32_t* cur = c->counts.h + (size_t)k * fg::K5_COUNT;
        const unsigned long long lo = d.encode ? c->enc_base.h[k] : 0, hi = d.encode ? c->enc_base.h[k + 1] : 0;
        d.overflow = d.overflow || tables_overflow(c, fmt, cur) || hi > c->enc_out_cap;
        if (d.overflow) continue;  // keep draining the events; the batch is redone
        if (!d.encode) {
            if (int rc = copy_tables_d2h(c, fmt, d.prev, cur, c->s_d2h)) return rc;
        } else if (hi > lo) {
            FG_CUDA(c, cudaMemcpyAsync(c->enc_out.h + lo, c->enc_out.d + lo, (size_t)(hi - lo), cudaMemcpyDeviceToHost, c->s_d2h));
        }
        d.prev = cur;
    }
    return FG_OK;
}

// drain_upto over the rest of `steps` parse steps.  total: the counters of the whole batch (the last snapshot).
int end_drain(fg_ctx* c, int fmt, int steps, Drain& d, uint32_t* total, bool& overflow) {
    if (int rc = drain_upto(c, fmt, steps, d)) return rc;
    overflow = d.overflow;
    memcpy(total, steps ? c->counts.h + (size_t)(steps - 1) * fg::K5_COUNT : kZeroCounts, kCountBytes);
    return FG_OK;
}

int drain(fg_ctx* c, int fmt, int steps, int encode, uint32_t* total, bool& overflow) {
    Drain d = begin_drain(c, encode);
    return end_drain(c, fmt, steps, d, total, overflow);
}

// End of an attempt of a pipelined call: waits for s_d2h, rejects a batch whose offsets failed the device check, and
// times the steps' kernels and the call so far
int finish(fg_ctx* c, int steps, const uint32_t* total, std::chrono::steady_clock::time_point t_begin, float& kernel_ms,
           float& total_ms) {
    FG_CUDA(c, cudaStreamSynchronize(c->s_d2h));
    if (total[fg::K5_BAD_OFFSETS]) return fail(c, FG_E_ARG, "offsets must be non-decreasing and within max_batch_bytes");
    if (total[fg::K5_LONG_JSON_SPAN])
        return fail(c, FG_E_CAPACITY, "a GELF string with escapes is too long to encode (GELF output: 1 GiB or more, LTSV output: 512 MiB or more)");
    kernel_ms = 0.f;
    for (int k = 0; k < steps; ++k) {
        float ms = 0.f;
        FG_CUDA(c, cudaEventElapsedTime(&ms, c->steps[k].k0, c->steps[k].k1));
        kernel_ms += ms;
    }
    total_ms = std::chrono::duration<float, std::milli>(std::chrono::steady_clock::now() - t_begin).count();
    return FG_OK;
}

// One pass over the resident batch on s_comp.  Only the counters below the bad-offsets word are zeroed: a failed
// fg_upload leaves that word set, which keeps the parse kernels inert.  `start`, when given, is recorded after the zeroing.
int resident_pass(fg_ctx* c, int fmt, int tile, cudaEvent_t start, bool time_dominant) {
    FG_CUDA(c, cudaMemsetAsync(c->k.d, 0, sizeof(uint32_t) * fg::K5_BAD_OFFSETS, c->s_comp));
    if (start) FG_CUDA(c, cudaEventRecord(start, c->s_comp));
    return launch_lines(c, fmt, 0, c->res_n, tile, nullptr, 0, c->s_comp, time_dominant);
}

// After the resident passes since ev_a: ev_b, the counter block, and unless a table overflowed, the time from ev_a to
// ev_b and the batch that fg_download returns
int resident_end(fg_ctx* c, int fmt, uint32_t* total, float* ms, bool& overflow) {
    FG_CUDA(c, cudaEventRecord(c->ev_b, c->s_comp));
    FG_CUDA(c, cudaMemcpyAsync(total, c->k.d, kCountBytes, cudaMemcpyDeviceToHost, c->s_comp));
    FG_CUDA(c, cudaStreamSynchronize(c->s_comp));
    overflow = tables_overflow(c, fmt, total);
    if (overflow) return FG_OK;
    float t = 0.f;
    FG_CUDA(c, cudaEventElapsedTime(&t, c->ev_a, c->ev_b));
    if (ms) *ms = t;
    c->res_fmt = fmt;
    memcpy(c->res_tot, total, kCountBytes);
    return FG_OK;
}

// serde_json 0.8 escape_bytes, for the keys / values of output.gelf_extra rendered once on the host
void json_escape_into(const std::string& v, std::string& o) {
    o.push_back('"');
    for (const char c : v) {
        switch (c) {
            case '"': o += "\\\""; break;
            case '\\': o += "\\\\"; break;
            case '\x08': o += "\\b"; break;
            case '\x0c': o += "\\f"; break;
            case '\n': o += "\\n"; break;
            case '\r': o += "\\r"; break;
            case '\t': o += "\\t"; break;
            default: o.push_back(c);
        }
    }
    o.push_back('"');
}

// The keys GelfEncoder::encode always or conditionally inserts (gelf_encoder.rs:60-100) merged with output.gelf_extra
// (:110-112, inserted last: an extra replaces a fixed key of the same name), sorted by key like the BTreeMap iterates.
int build_static_items(fg_ctx* c) {
    struct Item { std::string key, lit; int kind; };
    static const char* fixed[9] = {"application_name", "full_message", "host", "level", "process_id", "sd_id", "short_message",
                                   "timestamp", "version"};
    std::vector<Item> items;
    for (int k = 0; k < 9; ++k) {
        Item it;
        it.key = fixed[k];
        it.lit = ",";  // the device skips the comma for the first item of a record
        json_escape_into(it.key, it.lit);
        it.lit.push_back(':');
        it.kind = k;
        items.push_back(it);
    }
    for (const auto& kv : c->gelf_extra) {
        Item it;
        it.key = kv.first;
        it.lit = ",";
        json_escape_into(kv.first, it.lit);
        it.lit.push_back(':');
        json_escape_into(kv.second, it.lit);
        it.kind = 100;
        bool replaced = false;
        for (auto& x : items)
            if (x.key == it.key) { x = it; replaced = true; }
        if (!replaced) items.push_back(it);
    }
    std::sort(items.begin(), items.end(), [](const Item& a, const Item& b) { return a.key < b.key; });  // byte order (std::string compares as unsigned char)
    std::vector<int32_t> key_off{0}, lit_off, kind;
    std::string blob;
    for (const auto& it : items) {
        blob += it.key;
        key_off.push_back((int32_t)blob.size());
    }
    lit_off.push_back((int32_t)blob.size());
    for (const auto& it : items) {
        blob += it.lit;
        lit_off.push_back((int32_t)blob.size());
        kind.push_back(it.kind);
    }
    Packer p;
    p.add(blob);  // at offset 0: the key and literal offsets index the blob itself
    const size_t o_key = p.add(key_off), o_lit = p.add(lit_off), o_kind = p.add(kind);
    if (int rc = p.upload(c, c->static_blob)) return rc;
    const uint8_t* b = c->static_blob.d;
    c->n_static = (int)items.size();
    c->d_static_key_off = (const int32_t*)(b + o_key);
    c->d_static_lit_off = (const int32_t*)(b + o_lit);
    c->d_static_kind = (const int32_t*)(b + o_kind);
    return FG_OK;
}

int grow_enc_out(fg_ctx* c, size_t cap) {
    c->enc_out_cap = 0;
    cap = (cap + 4095) & ~(size_t)4095;
    FG_CUDA(c, c->enc_out.alloc(cap + 16, BOTH));
    c->enc_out_cap = cap;
    return FG_OK;
}

int ensure_encoder(fg_ctx* c, int fmt, int chunks) {
    const size_t L = (size_t)c->max_lines;
    if (fmt == FG_FMT_LTSV && !c->enc_stop.d) FG_CUDA(c, c->enc_stop.alloc(L, BOTH));
    if (!c->enc_lens.d) {
        FG_CUDA(c, c->enc_lens.alloc(L, DEV));
        FG_CUDA(c, c->enc_rel.alloc(L, DEV));
        FG_CUDA(c, c->enc_offsets.alloc(L + 1, BOTH));
        FG_CUDA(c, c->enc_status.alloc(L, BOTH));
        c->scan_temp_bytes = fg::gelf_scan_temp_bytes(c->max_lines);
        FG_CUDA(c, c->scan_temp.alloc(c->scan_temp_bytes + 256, DEV));
    }
    if (!c->enc_out_cap)
        if (int rc = grow_enc_out(c, c->max_bytes * 2 + L * 200)) return rc;
    if (c->enc_base.n < (size_t)chunks + 1) FG_CUDA(c, c->enc_base.alloc((size_t)chunks + 1, BOTH));
    if (!c->static_blob.d)
        if (int rc = build_static_items(c)) return rc;
    return FG_OK;
}

// After an overflow of a pipelined call: the allocators kept counting past the capacity, so each side table grows once to
// the exact need, and the encoder's output buffer too when `enc_need` (its size in bytes, 0 without the encoder) passes it
int regrow(fg_ctx* c, int fmt, const uint32_t* total, unsigned long long enc_need) {
    if (int rc = regrow_tables(c, fmt, total)) return rc;
    if (enc_need > c->enc_out_cap)
        if (int rc = grow_enc_out(c, (size_t)enc_need + (size_t)enc_need / 8 + 4096)) return rc;
    return FG_OK;
}

// End of a fused GELF call that encoded n records: its LTSV stops and wall clock become readable, and `out` points at
// its results
void end_fused(fg_ctx* c, int fmt, int32_t n, float kernel_ms, float total_ms, fg_encoded_out* out) {
    if (fmt == FG_FMT_LTSV) c->enc_stop_n = n;
    c->gelf_now_ok = fmt == FG_FMT_GELF;
    memset(out, 0, sizeof *out);
    out->n = n;
    out->bytes = c->enc_out.h;
    out->offsets = c->enc_offsets.h;
    out->status = c->enc_status.h;
    out->kernel_ms = kernel_ms;
    out->total_ms = total_ms;
}

// LTSVString::insert of every output.ltsv_extra pair (ltsv_encoder.rs:95-103: one leading '_' stripped from the key), each
// with the '\t' in front that the device drops for a record's first field: `\tkey:value...`
std::string ltsv_extra_literal(const std::vector<std::pair<std::string, std::string>>& kv) {
    std::string lit;
    for (const auto& [k0, v] : kv) {
        const std::string k = !k0.empty() && k0[0] == '_' ? k0.substr(1) : k0;
        lit.push_back('\t');
        for (const char ch : k) lit.push_back(ch == '\n' || ch == '\t' ? ' ' : (ch == ':' ? '_' : ch));
        lit.push_back(':');
        for (const char ch : v) lit.push_back(ch == '\n' || ch == '\t' ? ' ' : ch);
    }
    return lit;
}

// The caller's lines, framed already -> H2D and the parse kernels chunk_lines lines a step, and with `encode` the GELF
// encoder after each parse step: the pre-framed counterpart of split_stream, with the same results.  Without `encode`
// the rows and side tables come back, with it only the encoded records.  total, kernel_ms, total_ms: as drain and finish
// give them, zero for n == 0.
int batch_lines(fg_ctx* c, int fmt, const uint8_t* bytes, const int32_t* offsets, int32_t n, int encode, uint32_t* total,
                float& kernel_ms, float& total_ms) {
    if (int rc = begin_call(c, (fg_format)fmt)) return rc;
    const int C = c->chunk_lines;
    const int chunks = n > 0 ? (n + C - 1) / C : 1;
    if (encode)
        if (int rc = ensure_encoder(c, fmt, chunks)) return rc;
    if (n == 0) {
        if (encode) c->enc_offsets.h[0] = 0;
        memset(total, 0, kCountBytes);
        kernel_ms = total_ms = 0.f;
        return FG_OK;
    }
    const auto t_begin = std::chrono::steady_clock::now();
    HostBatch B{bytes, offsets, is_pinned(bytes), is_pinned(offsets), 0};
    if (int rc = ensure_steps(c, chunks)) return rc;
    const int tile = pick_tile(c, (size_t)(offsets[n] - offsets[0]), n, fmt);
    const int attempts = encode ? 3 : 2;  // encode: a side table and the output buffer may each overflow once
    for (int attempt = 0; attempt < attempts; ++attempt) {
        FG_CUDA(c, cudaMemsetAsync(c->k.d, 0, kCountBytes, c->s_comp));
        if (encode) FG_CUDA(c, cudaMemsetAsync(c->enc_base.d, 0, sizeof(unsigned long long), c->s_comp));
        B.bounce_ix = 0;
        for (int k = 0; k < chunks; ++k) {
            const int l0 = k * C, l1 = std::min(n, l0 + C);
            if (int rc = upload_chunk(c, B, k, l0, l1)) return rc;
            if (int rc = parse_step(c, fmt, k, l0, l1 - l0, tile, nullptr, 0, c->s_comp, encode)) return rc;
        }
        bool overflow;
        if (int rc = drain(c, fmt, chunks, encode, total, overflow)) return rc;
        if (int rc = finish(c, chunks, total, t_begin, kernel_ms, total_ms)) return rc;
        if (!overflow) return FG_OK;
        if (int rc = regrow(c, fmt, total, encode ? c->enc_base.h[chunks] : 0)) return rc;
    }
    return fail(c, FG_E_CAPACITY, encode ? "output / side table overflow after regrow" : "side table overflow after regrow");
}

// The Cap'n Proto encoder's refusal of a record it cannot hold: reset before the call, read after it.  capnp-rust asserts
// "Lists are limited to 2**29 elements" for a text of 2^29 - 1 bytes or more, so the reference writes no such message; the
// call fails and its output is not handed out.
int begin_capnp(fg_ctx* c, int enc) {
    if (enc != ENC_CAPNP) return FG_OK;
    FG_CUDA(c, cudaSetDevice(c->device));
    FG_CUDA(c, cudaMemset(c->k.d + kCapnpTooLong, 0xFF, sizeof(uint32_t)));
    return FG_OK;
}

// offsets [n + 1]: the batch's line offsets, which name the record the device reports by its first byte
int end_capnp(fg_ctx* c, int enc, const int32_t* offsets, int32_t n) {
    if (enc != ENC_CAPNP) return FG_OK;
    uint32_t at = 0;
    FG_CUDA(c, cudaMemcpy(&at, c->k.d + kCapnpTooLong, sizeof at, cudaMemcpyDeviceToHost));
    if (at == 0xFFFFFFFFu) return FG_OK;
    // the first line starting there that is not empty
    int32_t line = (int32_t)(std::lower_bound(offsets, offsets + n, (int32_t)at) - offsets);
    while (line + 1 < n && offsets[line + 1] == offsets[line]) ++line;
    const std::string what = "record " + std::to_string(line) + ": a text of 2^29 - 1 bytes or more does not fit a Cap'n Proto message";
    return fail(c, FG_E_ARG, what.c_str());
}

// decode + the encoder `enc` fused (fg_decode_encode_gelf / fg_decode_encode_ltsv)
int decode_encode(fg_ctx* c, int enc, fg_format fmt, const uint8_t* bytes, const int32_t* offsets, int32_t n, fg_encoded_out* out) {
    if (!c || !out) return FG_E_ARG;
    begin_fused(c, (int)fmt);
    if (int rc = check_batch(c, bytes, offsets, n)) return rc;
    if (int rc = check_fusable(c, (int)fmt)) return rc;
    uint32_t total[fg::K5_COUNT];
    float kms, tms;
    if (int rc = begin_capnp(c, enc)) return rc;
    if (int rc = batch_lines(c, (int)fmt, bytes, offsets, n, enc, total, kms, tms)) return rc;
    if (int rc = end_capnp(c, enc, offsets, n)) return rc;
    end_fused(c, (int)fmt, n, kms, tms, out);
    return FG_OK;
}

// everything fg_create sets up on the device
int init_device(fg_ctx* c, const fg_config* cfg) {
    FG_CUDA(c, cudaSetDevice(c->device));
    cudaDeviceProp prop;
    FG_CUDA(c, cudaGetDeviceProperties(&prop, c->device));
    const int max_tile = (int)std::min<size_t>(prop.sharedMemPerBlockOptin - 1024, 200 * 1024) & ~1023;
    c->num_sms = prop.multiProcessorCount;
    c->max_tile5 = (int)(((size_t)max_tile - 1024) * 8 / 9) & ~1023;  // tile + tile/8 bitmap + static shared memory
    FG_CUDA(c, fg::configure_kernels(c->max_tile5));
    FG_CUDA(c, create(c->s_h2d));
    FG_CUDA(c, create(c->s_comp));
    FG_CUDA(c, create(c->s_d2h));
    FG_CUDA(c, create(c->ev_a, cudaEventDefault));
    FG_CUDA(c, create(c->ev_b, cudaEventDefault));
    FG_CUDA(c, create(c->ev_dom0, cudaEventDefault));
    FG_CUDA(c, create(c->ev_dom1, cudaEventDefault));
    FG_CUDA(c, c->bytes.alloc(c->max_bytes + kPad, DEV));
    FG_CUDA(c, cudaMemset(c->bytes.d + c->max_bytes, 0, kPad));
    FG_CUDA(c, c->offsets.alloc((size_t)c->max_lines + 1, DEV));
    FG_CUDA(c, c->k.alloc(64, DEV));
    FG_CUDA(c, cudaMemset(c->k.d, 0, 256));
    for (int b = 0; b < 2; ++b) {
        FG_CUDA(c, c->bounce[b].alloc(kBounceBytes, HOST));
        FG_CUDA(c, create(c->bounce_ev[b], cudaEventDisableTiming));
    }
    return upload_ltsv_config(c, cfg);
}

}  // namespace

extern "C" {

int fg_create(const fg_config* cfg, fg_ctx** out) {
    if (!out) return FG_E_ARG;
    *out = nullptr;
    fg_config def{};
    if (!cfg) cfg = &def;
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) {
        cudaGetLastError();
        return FG_E_NO_DEVICE;  // no CPU fallback: the decoder does not exist without a GPU
    }
    if (cfg->device < 0 || cfg->device >= ndev) return FG_E_ARG;
    fg_ctx* c = new (std::nothrow) fg_ctx();
    if (!c) return FG_E_ARG;
    c->device = cfg->device;
    c->max_bytes = cfg->max_batch_bytes > 0 ? (size_t)cfg->max_batch_bytes : ((size_t)256 << 20);
    if (c->max_bytes > 0x7FFFFFC0ull) c->max_bytes = 0x7FFFFFC0ull;  // int32 offsets
    c->max_lines = cfg->max_batch_lines > 0 ? cfg->max_batch_lines : (2 << 20);
    c->max_lines = (c->max_lines + 63) & ~63;  // keeps every row column 256-byte aligned
    c->chunk_lines = cfg->chunk_lines > 0 ? cfg->chunk_lines : (512 << 10);
    c->chunk_lines = (c->chunk_lines + 127) / 128 * 128;  // a multiple of every kernel's lines per CTA
    c->r3164_year = cfg->rfc3164_year;
    c->input_format = cfg->input_format;
    if (cfg->tzdir) c->tzdir = cfg->tzdir;
    if (int rc = init_device(c, cfg)) {
        fprintf(stderr, "flowgger_cuda: %s\n", c->last_error.c_str());
        fg_destroy(c);
        return rc;
    }
    *out = c;
    return FG_OK;
}

void fg_destroy(fg_ctx* c) {
    if (!c) return;
    cudaSetDevice(c->device);
    cudaDeviceSynchronize();
    delete c;
}

const char* fg_last_error(const fg_ctx* c) { return c ? c->last_error.c_str() : "null context"; }

int fg_host_alloc(fg_ctx* c, size_t bytes, void** out) {
    if (!c || !out) return FG_E_ARG;
    FG_CUDA(c, cudaSetDevice(c->device));
    FG_CUDA(c, cudaHostAlloc(out, bytes ? bytes : 1, cudaHostAllocDefault));
    return FG_OK;
}
void fg_host_free(fg_ctx* c, void* p) {
    if (c && p) cudaFreeHost(p);
}

int fg_decode_batch(fg_ctx* c, fg_format fmt, const uint8_t* bytes, const int32_t* offsets, int32_t n,
                    fg_batch_out* out) {
    if (!c || !out) return FG_E_ARG;
    if (int rc = check_batch(c, bytes, offsets, n)) return rc;
    uint32_t total[fg::K5_COUNT];
    float kms, tms;
    if (int rc = batch_lines(c, (int)fmt, bytes, offsets, n, ENC_NONE, total, kms, tms)) return rc;
    memset(out, 0, sizeof *out);
    fill_out(c, fmt, n, total, out);
    out->kernel_ms = kms;
    out->total_ms = tms;
    return FG_OK;
}

int fg_set_rfc3164_year(fg_ctx* c, int32_t year) {
    if (!c) return FG_E_ARG;
    c->r3164_year = year;
    return FG_OK;
}

int fg_set_tz_table(fg_ctx* c, int32_t n_zones, const char* const* names, const int32_t* first, const int64_t* span_start_utc,
                    const int32_t* span_offset) {
    if (!c || n_zones < 0 || (n_zones > 0 && (!names || !first || !span_start_utc || !span_offset))) return FG_E_ARG;
    std::vector<std::string> nm;
    std::vector<fg::TzZoneSpans> zones;
    if (n_zones > 0 && first[0] < 0) return fail(c, FG_E_ARG, "fg_set_tz_table: first[] must start at a non-negative index");
    for (int32_t z = 0; z < n_zones; ++z) {
        const int32_t a = first[z], b = first[z + 1];
        if (!names[z] || !names[z][0] || b <= a) return fail(c, FG_E_ARG, "fg_set_tz_table: every zone needs a name and at least one span");
        fg::TzZoneSpans sp;
        for (int32_t j = a; j < b; ++j) {
            if (j > a) {
                if (j > a + 1 && span_start_utc[j] <= span_start_utc[j - 1]) return fail(c, FG_E_ARG, "fg_set_tz_table: span starts must ascend");
                sp.trans.push_back((long long)span_start_utc[j]);
            }
            sp.offs.push_back(span_offset[j]);
        }
        nm.emplace_back(names[z]);
        zones.push_back(std::move(sp));
    }
    FG_CUDA(c, cudaSetDevice(c->device));
    FG_CUDA(c, cudaDeviceSynchronize());
    fg::tz_build(nm, zones, c->tz_host);
    return upload_tz(c);
}

// host-side queries of the zone database (no device involved), for callers that want to check what a context will load
namespace {
std::mutex g_tz_mu;
std::string g_tz_dir;
fg::TzHostTable g_tz_table;
bool tz_query_table(const char* tzdir) {  // g_tz_mu held
    const std::string dir = tzdir ? tzdir : "";
    if (g_tz_table.loaded && dir == g_tz_dir) return true;
    std::string err;
    fg::TzHostTable t;
    if (!fg::tz_load_dir(tzdir, t, err)) return false;
    g_tz_table = std::move(t);
    g_tz_dir = dir;
    return true;
}
}  // namespace

// what get_by_name + assume_timezone answer for `name` at the local second `local`:
// 1 = found (offset stored), 0 = no such identifier, FG_E_ARG = the database could not be read
int fg_tz_lookup(const char* tzdir, const char* name, int64_t local, int32_t* offset) {
    if (!name) return FG_E_ARG;
    std::lock_guard<std::mutex> guard(g_tz_mu);
    if (!tz_query_table(tzdir)) return FG_E_ARG;
    const fg::TzDeviceTable T = g_tz_table.view();
    const int z = fg::tz_find(T, (const uint8_t*)name, 0, (int)strlen(name));
    if (z < 0) return 0;
    if (offset) *offset = fg::tz_offset_local(T, z, (long long)local);
    return 1;
}
// identifiers in the database under `tzdir` (negative: unreadable)
int32_t fg_tz_count(const char* tzdir) {
    std::lock_guard<std::mutex> guard(g_tz_mu);
    if (!tz_query_table(tzdir)) return FG_E_ARG;
    return (int32_t)g_tz_table.n_names();
}

int fg_set_gelf_extra(fg_ctx* c, int32_t n, const char* const* keys, const char* const* values) {
    if (!c || n < 0 || (n > 0 && (!keys || !values))) return FG_E_ARG;
    FG_CUDA(c, cudaSetDevice(c->device));
    c->gelf_extra.clear();
    for (int32_t k = 0; k < n; ++k) {
        if (!keys[k] || !values[k]) return fail(c, FG_E_ARG, "output.gelf_extra values must be strings");  // gelf_encoder.rs:41
        c->gelf_extra.emplace_back(keys[k], values[k]);
    }
    FG_CUDA(c, cudaDeviceSynchronize());
    return build_static_items(c);
}

int fg_set_output_framing(fg_ctx* c, fg_out_framing framing) {
    if (!c) return FG_E_ARG;
    if (framing != FG_OUT_NONE && framing != FG_OUT_LINE && framing != FG_OUT_NUL && framing != FG_OUT_SYSLEN)
        return fail(c, FG_E_ARG, "unknown output framing");
    c->out_framing = framing;
    return FG_OK;
}

// decode (RFC5424, RFC3164, LTSV or GELF) + GelfEncoder::encode fused: H2D lines -> parse kernels -> size / scan / write
// kernels -> D2H of the encoded records (and for LTSV the "Missing value" stops) only, chunk by chunk; the decoder's rows
// and side tables never leave the device.
int fg_decode_encode_gelf(fg_ctx* c, fg_format fmt, const uint8_t* bytes, const int32_t* offsets, int32_t n, fg_encoded_out* out) {
    return decode_encode(c, ENC_GELF, fmt, bytes, offsets, n, out);
}

// decode + LTSVEncoder::encode fused: the same pipeline with the LTSV encoder's kernels
int fg_decode_encode_ltsv(fg_ctx* c, fg_format fmt, const uint8_t* bytes, const int32_t* offsets, int32_t n, fg_encoded_out* out) {
    return decode_encode(c, ENC_LTSV, fmt, bytes, offsets, n, out);
}

int fg_set_ltsv_extra(fg_ctx* c, int32_t n, const char* const* keys, const char* const* values) {
    if (!c || n < 0 || (n > 0 && (!keys || !values))) return FG_E_ARG;
    std::vector<std::pair<std::string, std::string>> kv;
    for (int32_t k = 0; k < n; ++k) {
        if (!keys[k] || !values[k]) return fail(c, FG_E_ARG, "output.ltsv_extra values must be strings");  // ltsv_encoder.rs:22-24
        kv.emplace_back(keys[k], values[k]);
    }
    std::sort(kv.begin(), kv.end());  // a TOML table iterates its keys in byte order
    for (size_t k = 1; k < kv.size(); ++k)
        if (kv[k].first == kv[k - 1].first) return fail(c, FG_E_ARG, "output.ltsv_extra has a duplicate key");
    FG_CUDA(c, cudaSetDevice(c->device));
    FG_CUDA(c, cudaDeviceSynchronize());
    const std::string lit = ltsv_extra_literal(kv);
    Packer p;
    p.add(lit);
    if (int rc = p.upload(c, c->ltsv_extra)) return rc;
    c->ltsv_extra_len = (int)lit.size();
    return FG_OK;
}

// decode + CapnpEncoder::encode fused: the same pipeline with the Cap'n Proto encoder's kernels
int fg_decode_encode_capnp(fg_ctx* c, fg_format fmt, const uint8_t* bytes, const int32_t* offsets, int32_t n, fg_encoded_out* out) {
    return decode_encode(c, ENC_CAPNP, fmt, bytes, offsets, n, out);
}

int fg_set_capnp_extra(fg_ctx* c, int32_t n, const char* const* keys, const char* const* values) {
    if (!c || n < 0 || (n > 0 && (!keys || !values))) return FG_E_ARG;
    // A key or value of 2^29 - 1 bytes or more is a text capnp-rust asserts on in every record; the blob's bounds are
    // int32: both are refused here, before anything is copied, and the extras in use stay.
    const size_t text_at = (sizeof(int32_t) * (2 * (size_t)n + 1) + 15) & ~(size_t)15;
    size_t total = text_at;
    for (int32_t k = 0; k < n; ++k) {
        if (!keys[k] || !values[k]) return fail(c, FG_E_ARG, "output.capnp_extra values must be strings");  // capnp_encoder.rs:25-27
        const size_t kl = strlen(keys[k]), vl = strlen(values[k]);
        if (kl + 1 >= fg::kCapMaxWords || vl + 1 >= fg::kCapMaxWords)
            return fail(c, FG_E_ARG, "output.capnp_extra: a key or value of 2^29 - 1 bytes or more does not fit a Cap'n Proto message");
        total += kl + vl;
        if (total > (size_t)INT32_MAX) return fail(c, FG_E_ARG, "output.capnp_extra: more than 2^31 - 1 bytes in all");
    }
    std::vector<std::pair<std::string, std::string>> kv;
    for (int32_t k = 0; k < n; ++k) kv.emplace_back(keys[k], values[k]);
    std::sort(kv.begin(), kv.end());  // a TOML table iterates its keys in byte order
    for (size_t k = 1; k < kv.size(); ++k)
        if (kv[k].first == kv[k - 1].first) return fail(c, FG_E_ARG, "output.capnp_extra has a duplicate key");
    FG_CUDA(c, cudaSetDevice(c->device));
    FG_CUDA(c, cudaDeviceSynchronize());
    // one blob: the bounds, then the text they index from the blob's start (the bounds take 2n + 1 words, padded to 16 bytes)
    std::string text;
    std::vector<int32_t> off{(int32_t)text_at};
    for (const auto& [k, v] : kv) {
        text += k;
        off.push_back((int32_t)(text_at + text.size()));
        text += v;
        off.push_back((int32_t)(text_at + text.size()));
    }
    Packer p;
    p.add(off);
    p.add(text);
    if (int rc = p.upload(c, c->capnp_extra)) return rc;
    c->d_capnp_extra_off = (const int32_t*)c->capnp_extra.d;
    c->capnp_extra_n = (int)kv.size();
    return FG_OK;
}

// decode + PassthroughEncoder::encode fused: the same pipeline with the passthrough encoder's kernels
int fg_decode_encode_passthrough(fg_ctx* c, fg_format fmt, const uint8_t* bytes, const int32_t* offsets, int32_t n, fg_encoded_out* out) {
    return decode_encode(c, ENC_PASSTHROUGH, fmt, bytes, offsets, n, out);
}

int fg_set_passthrough_prefix(fg_ctx* c, const uint8_t* bytes, int64_t n) {
    if (!c || n < 0) return FG_E_ARG;
    if (n > 0 && !bytes) return fail(c, FG_E_ARG, "passthrough prefix: NULL bytes");
    if (n > (int64_t)INT32_MAX) return fail(c, FG_E_ARG, "passthrough prefix: 2^31 bytes or more");
    FG_CUDA(c, cudaSetDevice(c->device));
    FG_CUDA(c, cudaDeviceSynchronize());
    c->pt_prefix_len = 0;
    // set once per call by the host layers (the header carries the time): the buffer is kept while the header fits
    if (c->pt_prefix.n < (size_t)n + 16) FG_CUDA(c, c->pt_prefix.alloc((size_t)n + 16, DEV));
    if (n > 0) FG_CUDA(c, cudaMemcpy(c->pt_prefix.d, bytes, (size_t)n, cudaMemcpyHostToDevice));
    c->pt_prefix_len = (int32_t)n;
    return FG_OK;
}

int fg_encoded_ltsv_stops(const fg_ctx* c, const int32_t** stop) {
    if (!c || !stop || c->enc_stop_n < 0) return FG_E_ARG;
    *stop = c->enc_stop.h;
    return FG_OK;
}

int fg_encoded_gelf_now(const fg_ctx* c, double* now) {
    if (!c || !now || !c->gelf_now_ok) return FG_E_ARG;
    *now = c->gelf_now;
    return FG_OK;
}

}  // extern "C"

namespace {

// Raw stream -> framing + UTF-8 check (split kernels on s_comp, 64 MiB chunk by chunk) -> parse kernels on s_parse,
// and with `encode` the GELF encoder after each parse step.  Without `encode` the rows and side tables come back, with
// it only the encoded records; the line offsets come back into split_offsets.h either way.  n: records framed; total,
// kernel_ms, total_ms: as drain and finish give them.
int split_stream(fg_ctx* c, int fmt, fg_framing framing, const uint8_t* stream, int64_t nbytes, int encode, int32_t& n,
                 uint32_t* total, float& kernel_ms, float& total_ms) {
    if (framing != FG_FRAME_LINE && framing != FG_FRAME_NUL) return fail(c, FG_E_ARG, "unknown framing");
    const int delim = framing == FG_FRAME_NUL ? 0 : '\n';
    const int strip = framing == FG_FRAME_NUL ? 2 : 1;
    if (nbytes < 0 || (nbytes > 0 && !stream)) return fail(c, FG_E_ARG, "null input");
    if ((size_t)nbytes > c->max_bytes) return fail(c, FG_E_CAPACITY, "stream has more bytes than max_batch_bytes");
    if (int rc = begin_call(c, (fg_format)fmt)) return rc;
    const auto t_begin = std::chrono::steady_clock::now();
    constexpr long long kChunk = 64ll << 20;  // pipeline granularity in bytes (a multiple of the 8 KB framing segment)
    const int chunks = nbytes > 0 ? (int)((nbytes + kChunk - 1) / kChunk) : 1;
    if (encode)
        if (int rc = ensure_encoder(c, fmt, chunks)) return rc;  // at most one parse step per chunk
    if (!c->seg.d) {
        FG_CUDA(c, c->seg.alloc((size_t)fg::split_segments((long long)c->max_bytes) + 16, DEV));
        FG_CUDA(c, c->n_lines.alloc(64, BOTH));
        FG_CUDA(c, c->invalid.alloc((size_t)c->max_lines + 64, DEV));
        FG_CUDA(c, c->split_offsets.alloc((size_t)c->max_lines + 1, HOST));
        FG_CUDA(c, create(c->ev_s0, cudaEventDefault));
        FG_CUDA(c, create(c->ev_s1, cudaEventDefault));
        FG_CUDA(c, create(c->s_parse));
    }
    if ((int)c->ev_split.size() < chunks + 1) {
        const size_t want = (size_t)chunks + 1;
        while (c->ev_split.size() < want) {
            Event e;
            FG_CUDA(c, create(e, cudaEventDisableTiming));
            c->ev_split.push_back(std::move(e));
        }
        FG_CUDA(c, c->cum.alloc(want, BOTH));
    }
    if (int rc = ensure_steps(c, chunks + 1)) return rc;
    const bool pinned = nbytes > 0 && is_pinned(stream);

    const int attempts = encode ? 3 : 2;  // encode: a side table and the output buffer may each overflow once
    for (int attempt = 0; attempt < attempts; ++attempt) {
        // ---- enqueue, chunk by chunk: raw bytes -> HBM, then framing + UTF-8 validation of that chunk (no host dependency)
        FG_CUDA(c, cudaMemsetAsync(c->n_lines.d + 8, 0, 4, c->s_comp));  // running newline count (uint32 at n_lines[8])
        FG_CUDA(c, cudaMemsetAsync(c->invalid.d, 0, (size_t)c->max_lines, c->s_comp));
        FG_CUDA(c, cudaMemsetAsync(c->k.d, 0, kCountBytes, c->s_comp));
        if (encode) FG_CUDA(c, cudaMemsetAsync(c->enc_base.d, 0, sizeof(unsigned long long), c->s_comp));
        FG_CUDA(c, cudaEventRecord(c->ev_s0, c->s_comp));
        int bounce_ix = 0;
        for (int k = 0; k < chunks; ++k) {
            const long long c0 = (long long)k * kChunk, c1 = std::min<long long>(nbytes, c0 + kChunk);
            const bool last = k == chunks - 1;
            if (int rc = h2d(c, c->bytes.d + c0, stream + c0, (size_t)(c1 - c0), pinned, bounce_ix)) return rc;
            if (last) FG_CUDA(c, cudaMemsetAsync(c->bytes.d + nbytes, delim ? 0 : 0xFF, 64, c->s_h2d));  // whole-vector loads past the end see no delimiter
            FG_CUDA(c, cudaEventRecord(c->steps[k].h2d, c->s_h2d));
            FG_CUDA(c, cudaStreamWaitEvent(c->s_comp, c->steps[k].h2d, 0));
            FG_CUDA(c, fg::launch_split_chunk(c->bytes.d, (long long)nbytes, c0, c1, last ? 1 : 0, c->seg.d, (uint32_t*)(c->n_lines.d + 8),
                                              c->cum.d + k, c->offsets.d, c->n_lines.d, c->max_lines, c->invalid.d, delim, c->s_comp));
            c->launches += 4;
            FG_CUDA(c, cudaMemcpyAsync(c->cum.h + k, c->cum.d + k, 4, cudaMemcpyDeviceToHost, c->s_comp));
            if (last) {
                FG_CUDA(c, cudaMemcpyAsync(c->n_lines.h, c->n_lines.d, 4, cudaMemcpyDeviceToHost, c->s_comp));
                FG_CUDA(c, cudaEventRecord(c->ev_s1, c->s_comp));
            }
            FG_CUDA(c, cudaEventRecord(c->ev_split[k], c->s_comp));
        }
        // ---- parse the lines that END in chunk k once chunk k+1 has been validated too (a sequence that starts in the
        //      last 16 bytes of a chunk is checked with the next one); what a step produced goes back while later chunks
        //      are still in flight
        int32_t done_lines = 0;
        n = 0;
        int nparse = 0;
        bool over = false;
        Drain d = begin_drain(c, encode);
        for (int k = 0; k < chunks; ++k) {
            const int dep = std::min(k + 1, chunks - 1);
            FG_CUDA(c, cudaEventSynchronize(c->ev_split[dep]));
            int32_t upto = c->cum.h[k];
            if (upto < 0) { over = true; break; }
            if (k == chunks - 1) {
                n = *c->n_lines.h;
                if (n < 0) { over = true; break; }
                upto = n;  // includes an unterminated last line
            }
            const int32_t cnt = upto - done_lines;
            if (cnt > 0) {
                const size_t span_bytes = (size_t)std::min<long long>(nbytes, (long long)(k + 1) * kChunk) - (size_t)((long long)k * kChunk);
                const int tile = pick_tile(c, std::max<size_t>(span_bytes, 1), cnt, (int)fmt);
                FG_CUDA(c, cudaStreamWaitEvent(c->s_parse, c->ev_split[dep], 0));
                if (int rc = parse_step(c, fmt, nparse, done_lines, cnt, tile, c->invalid.d + done_lines, strip, c->s_parse, encode)) return rc;
                ++nparse;
                done_lines = upto;
                if (int rc = drain_upto(c, fmt, nparse - 1, d)) return rc;  // the step before this one
            }
        }
        if (over) {
            FG_CUDA(c, cudaDeviceSynchronize());
            return fail(c, FG_E_CAPACITY, "stream has more lines than max_batch_lines");
        }
        // ---- the last step, line offsets
        bool overflow;
        if (int rc = end_drain(c, fmt, nparse, d, total, overflow)) return rc;
        if (!overflow)
            FG_CUDA(c, cudaMemcpyAsync(c->split_offsets.h, c->offsets.d, sizeof(int32_t) * ((size_t)n + 1), cudaMemcpyDeviceToHost, c->s_d2h));
        if (int rc = finish(c, nparse, total, t_begin, kernel_ms, total_ms)) return rc;
        if (overflow) {
            if (int rc = regrow(c, fmt, total, encode ? c->enc_base.h[nparse] : 0)) return rc;
            continue;
        }
        FG_CUDA(c, cudaEventElapsedTime(&c->last_split_ms, c->ev_s0, c->ev_s1));  // includes waiting for the H2D chunks
        if (encode && nparse == 0) c->enc_offsets.h[0] = 0;
        return FG_OK;
    }
    return fail(c, FG_E_CAPACITY, encode ? "output / side table overflow after regrow" : "side table overflow after regrow");
}

// framing + decode + the encoder `enc` fused (fg_split_decode_encode_gelf / fg_split_decode_encode_ltsv)
int split_decode_encode(fg_ctx* c, int enc, fg_format fmt, fg_framing framing, const uint8_t* stream, int64_t nbytes,
                        fg_encoded_out* out, const int32_t** line_offsets) {
    if (!c || !out || !line_offsets) return FG_E_ARG;
    begin_fused(c, (int)fmt);
    if (int rc = check_fusable(c, (int)fmt)) return rc;
    int32_t n;
    uint32_t total[fg::K5_COUNT];
    float kms, tms;
    if (int rc = begin_capnp(c, enc)) return rc;
    if (int rc = split_stream(c, (int)fmt, framing, stream, nbytes, enc, n, total, kms, tms)) return rc;
    if (int rc = end_capnp(c, enc, c->split_offsets.h, n)) return rc;
    end_fused(c, (int)fmt, n, kms, tms, out);
    *line_offsets = c->split_offsets.h;
    return FG_OK;
}

}  // namespace

extern "C" {

int fg_split_decode(fg_ctx* c, fg_format fmt, const uint8_t* stream, int64_t nbytes, fg_batch_out* out) {
    return fg_split_decode_framed(c, fmt, FG_FRAME_LINE, stream, nbytes, out);
}

int fg_split_decode_framed(fg_ctx* c, fg_format fmt, fg_framing framing, const uint8_t* stream, int64_t nbytes, fg_batch_out* out) {
    if (!c || !out) return FG_E_ARG;
    if ((int)fmt < 0 || (int)fmt > 3) return fail(c, FG_E_ARG, "unknown format");
    int32_t n;
    uint32_t total[fg::K5_COUNT];
    float kms, tms;
    if (int rc = split_stream(c, (int)fmt, framing, stream, nbytes, ENC_NONE, n, total, kms, tms)) return rc;
    memset(out, 0, sizeof *out);
    fill_out(c, fmt, n, total, out);
    out->line_offsets = c->split_offsets.h;
    out->kernel_ms = kms;
    out->total_ms = tms;
    return FG_OK;
}

// framing + decode (RFC5424, RFC3164, LTSV or GELF) + GelfEncoder::encode on the device: only the encoded records, the line
// offsets and for LTSV the "Missing value" stops come back
int fg_split_decode_encode_gelf(fg_ctx* c, fg_format fmt, fg_framing framing, const uint8_t* stream, int64_t nbytes, fg_encoded_out* out,
                                const int32_t** line_offsets) {
    return split_decode_encode(c, ENC_GELF, fmt, framing, stream, nbytes, out, line_offsets);
}

// framing + decode + LTSVEncoder::encode on the device, as fg_split_decode_encode_gelf
int fg_split_decode_encode_ltsv(fg_ctx* c, fg_format fmt, fg_framing framing, const uint8_t* stream, int64_t nbytes, fg_encoded_out* out,
                                const int32_t** line_offsets) {
    return split_decode_encode(c, ENC_LTSV, fmt, framing, stream, nbytes, out, line_offsets);
}

// framing + decode + CapnpEncoder::encode on the device, as fg_split_decode_encode_gelf
int fg_split_decode_encode_capnp(fg_ctx* c, fg_format fmt, fg_framing framing, const uint8_t* stream, int64_t nbytes, fg_encoded_out* out,
                                 const int32_t** line_offsets) {
    return split_decode_encode(c, ENC_CAPNP, fmt, framing, stream, nbytes, out, line_offsets);
}

// framing + decode + PassthroughEncoder::encode on the device, as fg_split_decode_encode_gelf
int fg_split_decode_encode_passthrough(fg_ctx* c, fg_format fmt, fg_framing framing, const uint8_t* stream, int64_t nbytes,
                                       fg_encoded_out* out, const int32_t** line_offsets) {
    return split_decode_encode(c, ENC_PASSTHROUGH, fmt, framing, stream, nbytes, out, line_offsets);
}

int fg_upload(fg_ctx* c, const uint8_t* bytes, const int32_t* offsets, int32_t n) {
    if (int rc = check_batch(c, bytes, offsets, n)) return rc;
    FG_CUDA(c, cudaSetDevice(c->device));
    if (n > 0) {
        const size_t b0 = (size_t)offsets[0], b1 = (size_t)offsets[n];
        FG_CUDA(c, cudaMemcpy(c->bytes.d + b0, bytes + b0, b1 - b0, cudaMemcpyHostToDevice));
        FG_CUDA(c, cudaMemcpy(c->offsets.d, offsets, sizeof(int32_t) * ((size_t)n + 1), cudaMemcpyHostToDevice));
        c->res_bytes = b1 - b0;
    } else {
        c->res_bytes = 0;
    }
    FG_CUDA(c, cudaMemset(c->k.d, 0, kCountBytes));
    FG_CUDA(c, fg::launch_check_offsets(c->offsets.d, n, (long long)c->max_bytes, c->k.d + fg::K5_BAD_OFFSETS, c->s_comp));
    uint32_t bad = 0;
    FG_CUDA(c, cudaMemcpyAsync(&bad, c->k.d + fg::K5_BAD_OFFSETS, 4, cudaMemcpyDeviceToHost, c->s_comp));
    FG_CUDA(c, cudaStreamSynchronize(c->s_comp));
    if (bad) return fail(c, FG_E_ARG, "offsets must be non-decreasing and within max_batch_bytes");
    c->res_n = n;
    c->res_fmt = -1;
    return FG_OK;
}

int fg_parse_resident(fg_ctx* c, fg_format fmt, float* kernel_ms) {
    if (!c) return FG_E_ARG;
    if (int rc = begin_call(c, fmt)) return rc;
    for (int attempt = 0; attempt < 2; ++attempt) {
        if (int rc = resident_pass(c, (int)fmt, pick_tile(c, c->res_bytes, c->res_n, (int)fmt), c->ev_a, true)) return rc;
        uint32_t total[fg::K5_COUNT] = {};
        bool overflow;
        if (int rc = resident_end(c, (int)fmt, total, kernel_ms, overflow)) return rc;
        if (overflow) {
            if (int rc = regrow_tables(c, (int)fmt, total)) return rc;
            continue;
        }
        FG_CUDA(c, cudaEventElapsedTime(&c->last_dom_ms, c->ev_dom0, c->ev_dom1));
        return FG_OK;
    }
    return fail(c, FG_E_CAPACITY, "side table overflow after regrow");
}

// K back-to-back passes over the resident batch with ONE host synchronisation at the end (what bench.py times):
// total_ms = CUDA-event time from before the first launch to after the last one.
int fg_parse_resident_n(fg_ctx* c, fg_format fmt, int32_t k, float* total_ms) {
    if (!c || k < 1) return FG_E_ARG;
    if (int rc = begin_call(c, fmt)) return rc;
    // the side tables must already be large enough (one fg_parse_resident warm-up regrows them): checked after the loop
    const int tile = pick_tile(c, c->res_bytes, c->res_n, (int)fmt);
    FG_CUDA(c, cudaEventRecord(c->ev_a, c->s_comp));
    for (int32_t it = 0; it < k; ++it)
        if (int rc = resident_pass(c, (int)fmt, tile, nullptr, false)) return rc;
    uint32_t total[fg::K5_COUNT] = {};
    bool overflow;
    if (int rc = resident_end(c, (int)fmt, total, total_ms, overflow)) return rc;
    if (overflow) return fail(c, FG_E_CAPACITY, "side table too small: call fg_parse_resident once before fg_parse_resident_n");
    return FG_OK;
}

int fg_download(fg_ctx* c, fg_format fmt, fg_batch_out* out) {
    if (!c || !out) return FG_E_ARG;
    if (c->res_fmt != (int)fmt) return fail(c, FG_E_ARG, "no resident parse of this format to download");
    FG_CUDA(c, cudaSetDevice(c->device));
    memset(out, 0, sizeof *out);
    const uint32_t zero[fg::K5_COUNT] = {};
    if (int rc = copy_rows_d2h(c, fmt, 0, c->res_n, c->s_d2h)) return rc;
    if (int rc = copy_tables_d2h(c, (int)fmt, zero, c->res_tot, c->s_d2h)) return rc;
    FG_CUDA(c, cudaStreamSynchronize(c->s_d2h));
    fill_out(c, fmt, c->res_n, c->res_tot, out);
    return FG_OK;
}

int fg_flush_l2(fg_ctx* c) {
    if (!c) return FG_E_ARG;
    FG_CUDA(c, cudaSetDevice(c->device));
    if (!c->flush.d) FG_CUDA(c, c->flush.alloc(kL2FlushBytes, DEV));
    FG_CUDA(c, cudaMemsetAsync(c->flush.d, 0x5A, kL2FlushBytes, c->s_comp));
    FG_CUDA(c, cudaStreamSynchronize(c->s_comp));
    return FG_OK;
}

const char* fg_error_string(fg_format, uint32_t status) {
    if (status == FG_EP_NO_RAW) return "Cannot output empty raw message";  // encoder/passthrough_encoder.rs:44
    if (status == 0 || status >= FG_ST_COUNT) return nullptr;
    return kErrorStrings[status];
}
uint32_t fg_error_count(void) { return FG_ST_COUNT; }

const char* fg_build_info(void) { return fg::kernel_build_info(); }
int64_t fg_kernel_launches(const fg_ctx* c) { return c ? c->launches : 0; }
float fg_last_split_ms(const fg_ctx* c) { return c ? c->last_split_ms : 0.f; }
float fg_last_dominant_kernel_ms(const fg_ctx* c) { return c ? c->last_dom_ms : 0.f; }

}  // extern "C"
