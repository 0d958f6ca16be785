/* flowgger_cuda.h — C ABI of the H100 batched log-line decoder.
 *
 * Drop-in boundary for flowgger's Decoder stage.  The reference interface this
 * replaces is
 *     trait Decoder { fn decode(&self, line: &str) -> Result<Record, &'static str>; }
 *         (flowgger src/flowgger/decoder/mod.rs:44-46)
 * constructed by RFC5424Decoder::new / LTSVDecoder::new / GelfDecoder::new / RFC3164Decoder::new
 *         (decoder/rfc5424_decoder.rs:12, ltsv_decoder.rs:24, gelf_decoder.rs:16, rfc3164_decoder.rs:14)
 * and called once per record by the splitters
 *         (splitter/line_splitter.rs:50, nul_splitter.rs:57, syslen_splitter.rs:65).
 * The batched form is: N lines packed into one contiguous byte buffer plus an
 * int32 offsets array -> one fg_decode_batch() call -> N columnar results
 * (status code == the reference's Err(&'static str), or the Record fields as
 * zero-copy spans into the caller's byte buffer plus normalised scalars; escaped
 * RFC5424 SD values are unescaped on the device into a small arena).
 *
 * Plain C: pointers and sizes only.  No CPU fallback exists behind this ABI:
 * every entry point that parses runs the sm_90a CUDA kernels or fails.
 */
#ifndef FLOWGGER_CUDA_H
#define FLOWGGER_CUDA_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* input.format (mod.rs:413-422) */
typedef enum fg_format { FG_FMT_RFC5424 = 0, FG_FMT_LTSV = 1, FG_FMT_GELF = 2, FG_FMT_RFC3164 = 3 } fg_format;

/* SDValue discriminant (record.rs:4-11) + table-internal marker */
typedef enum fg_tag {
    FG_TAG_STRING = 0,
    FG_TAG_BOOL = 1,
    FG_TAG_F64 = 2,
    FG_TAG_I64 = 3,
    FG_TAG_U64 = 4,
    FG_TAG_NULL = 5,
    FG_TAG_SD_HEADER = 7 /* entry opens a StructuredData element: name = sd_id, val = #pairs */
} fg_tag;

/* entry_meta bits */
#define FG_EM_TAG_MASK 0x07u
#define FG_EM_UNESCAPE 0x08u  /* string value holds escapes: RFC5424 (rfc5424_decoder.rs:105-125) or JSON */
#define FG_EM_NO_PREFIX 0x10u /* GELF: name already starts with '_' (gelf_decoder.rs:99-103); else host prepends "_" */
#define FG_EM_SUFFIX 0x20u    /* LTSV: append the configured type suffix (ltsv_decoder.rs:131-136) */
#define FG_EM_NAME_ESC 0x40u  /* GELF: name span holds JSON escapes */
#define FG_EM_ARENA 0x80u     /* string value: off indexes fg_batch_out.arena (already unescaped), not `bytes` */

/* row meta word: status | facility<<8 | severity<<16 | flags<<24 */
#define FG_META_STATUS(m) ((uint32_t)(m)&0xFFu)
#define FG_META_FACILITY(m) (((uint32_t)(m) >> 8) & 0xFFu) /* 0xFF = None */
#define FG_META_SEVERITY(m) (((uint32_t)(m) >> 16) & 0xFFu) /* 0xFF = None */
#define FG_META_FLAGS(m) (((uint32_t)(m) >> 24) & 0xFFu)
#define FG_FLAG_TS_MISSING 0x01u   /* GELF without "timestamp": host fills wall clock (gelf_decoder.rs:109) */
#define FG_FLAG_MISSING_VALUE 0x02u /* LTSV part without ':' seen (println! at ltsv_decoder.rs:99) */
#define FG_FLAG_HOST_ESC 0x04u     /* GELF: hostname span holds JSON escapes */
#define FG_FLAG_MSG_ESC 0x08u      /* GELF: short_message span holds JSON escapes */
#define FG_FLAG_FULL_ESC 0x10u     /* GELF: full_message span holds JSON escapes */
#define FG_FLAG_NL_RETRY 0x20u     /* GELF: parsed through the raw-newline retry (gelf_decoder.rs:44-46) */
#define FG_FLAG_MSG_ARENA 0x40u    /* RFC3164: msg.off indexes fg_batch_out.arena — the message tokens re-joined by single
                                      spaces on the device (rfc3164_decoder.rs:67); without the flag the re-joined message is
                                      a span of the input */
#define FG_FLAG_WIDE 0x80u         /* RFC5424: the row lives in fg_batch_out.wide_rows[row.sd_first] (unusual shape, line >= 64 KiB, ...) */

/* (offset,len) into the `bytes` buffer given to the call; off < 0 => None */
typedef struct fg_span {
    int32_t off;
    int32_t len;
} fg_span;

/* ---- RFC5424 results are COMPACT: 32 bytes per line + 8 bytes per structured-data row -------------------------
 * All positions are u16 byte offsets relative to the start of the line.  Lines that are valid but not of the regular
 * shape `<PRI>1 TS HOST APP PROCID MSGID (-|[id name="value" ...]...) MSG` (a BOM, a delimiter-class byte inside a
 * header field, stray quotes ...) or are 64 KiB or longer are flagged FG_FLAG_WIDE and delivered as fg_wide_row
 * instead; they are decoded by the slow, exact kernel.  The header fields of RFC5424 are
 * consecutive (rfc5424_decoder.rs:23-30), so five space positions give hostname / appname / procid / msgid:
 *     hostname = [sp[0]+1, sp[1])   appname = [sp[1]+1, sp[2])   procid = [sp[2]+1, sp[3])   msgid = [sp[3]+1, sp[4])
 *     msg      = msg_len ? [msg_off, msg_off+msg_len) : None
 *     full_msg = [0, end)  with end = msg_len ? msg_off+msg_len : msg_off
 * Error rows (status != 0) carry only `meta`.  fg_row5424_* below decode a row into spans of the caller's buffer. */
typedef struct fg_row5424 {
    double ts;          /* Record.ts, bit-exact */
    uint32_t meta;      /* FG_META_* */
    uint32_t sd_first;  /* first row of this line in entries8 (FG_FLAG_WIDE: index into wide_rows) */
    uint16_t sd_count;  /* rows of this line in entries8; 0 => Record.sd = None */
    uint16_t sp[5];     /* positions of the 2nd .. 6th space */
    uint16_t msg_off;
    uint16_t msg_len;
} fg_row5424;

/* entries8 rows (uint64), positions relative to the line start; bits 63..62 select the kind:
 *   FG_E8_HEADER : sd_id start | sd_id end << 16 | #pairs << 32        opens a StructuredData element
 *   (neither)    : name start | name end << 16 | value end << 32      value = [name end + 2, value end), no escapes
 *   FG_E8_ARENA  : name start | name end << 16 | (arena offset / 2) << 32
 *                  the value held escapes and was unescaped on the device (rfc5424_decoder.rs:105-125): the record at
 *                  that offset of fg_batch_out.arena is [uint16 length][bytes] */
#define FG_E8_HEADER (1ull << 63)
#define FG_E8_ARENA (1ull << 62)
#define FG_E8_ARENA_OFF(e) ((uint32_t)(((e) >> 32) & 0x3FFFFFFFu) << 1)
#define FG_E8_A(e) ((uint32_t)((e)&0xFFFFu))
#define FG_E8_B(e) ((uint32_t)(((e) >> 16) & 0xFFFFu))
#define FG_E8_C(e) ((uint32_t)(((e) >> 32) & 0xFFFFu))

/* a line the compact row cannot hold: absolute spans like the LTSV / GELF columns; its structured data are rows
 * [sd.off, sd.off+sd.len) of entry_name / entry_val / entry_meta */
typedef struct fg_wide_row {
    int32_t line;
    uint32_t meta;
    double ts;
    fg_span hostname, appname, procid, msgid, msg, full_msg, sd;
} fg_wide_row;

static inline fg_span fg_row5424_field(const fg_row5424* r, int32_t line_off, int k /* 0 host, 1 app, 2 procid, 3 msgid */) {
    fg_span s;
    s.off = line_off + (int32_t)r->sp[k] + 1;
    s.len = (int32_t)r->sp[k + 1] - (int32_t)r->sp[k] - 1;
    return s;
}
static inline fg_span fg_row5424_msg(const fg_row5424* r, int32_t line_off) {
    fg_span s;
    s.off = r->msg_len ? line_off + (int32_t)r->msg_off : -1;
    s.len = (int32_t)r->msg_len;
    return s;
}
static inline fg_span fg_row5424_full(const fg_row5424* r, int32_t line_off) {
    fg_span s;
    s.off = line_off;
    s.len = (int32_t)r->msg_off + (int32_t)r->msg_len;
    return s;
}

/* LTSV schema value types (ltsv_decoder.rs:36-43) */
typedef enum fg_ltsv_type { FG_LTSV_STRING = 0, FG_LTSV_BOOL = 1, FG_LTSV_F64 = 2, FG_LTSV_I64 = 3, FG_LTSV_U64 = 4 } fg_ltsv_type;

typedef struct fg_config {
    int32_t device;           /* CUDA device ordinal */
    int64_t max_batch_bytes;  /* capacity of one fg_decode_batch call (<= 2^31-64) ; 0 = default 256 MiB */
    int32_t max_batch_lines;  /* 0 = default 2 Mi (rounded up to a multiple of 64) */
    int32_t chunk_lines;      /* host<->device pipeline granularity; 0 = default 256 Ki */
    /* input.ltsv_schema / input.ltsv_suffixes (ltsv_decoder.rs:25-81); ignored by other formats */
    int32_t ltsv_has_schema;
    int32_t ltsv_schema_len;
    const char* const* ltsv_schema_names; /* NUL-terminated UTF-8 */
    const int32_t* ltsv_schema_types;     /* fg_ltsv_type */
    const char* ltsv_suffix[5];           /* indexed by fg_ltsv_type; NULL = none ([0] unused) */
    /* input.format = "rfc3164": the two things RFC3164Decoder takes from its environment.
     * rfc3164_year: the year a timestamp without one belongs to — `OffsetDateTime::now_utc().year()`,
     *   rfc3164_decoder.rs:175.  0 = the UTC year of the clock at each fg_decode_batch / fg_split_decode call.
     * tzdir: directory of TZif files (RFC 8536) behind `time_tz::timezones::get_by_name`, :196.  NULL = $TZDIR, else
     *   /usr/share/zoneinfo.  Read on the first RFC3164 call; fg_set_tz_table replaces it with the caller's own table. */
    int32_t rfc3164_year;
    const char* tzdir;
    /* input.format the context is created for (mod.rs:413-422: the reference builds one decoder per configuration);
     * 0 = rfc5424.  Decoding takes the format per call; the fused GELF encoder takes LTSV input only on a context created
     * for LTSV, because it writes the pair keys with that context's ltsv_suffixes. */
    int32_t input_format;
} fg_config;

/* Columnar result of one batch.  All pointers are host pointers owned by the
 * context, valid until the next fg_decode_batch / fg_destroy on it. */
typedef struct fg_batch_out {
    int32_t n;         /* lines */
    int32_t n_entries; /* rows of the structured-data side table */
    const double* ts;        /* Record.ts (record.rs:72); utils/mod.rs:24-28 arithmetic, bit-exact */
    const uint32_t* meta;    /* FG_META_* */
    const fg_span* hostname; /* Record.hostname */
    const fg_span* appname;  /* RFC5424 only, else NULL */
    const fg_span* procid;   /* RFC5424 only, else NULL */
    const fg_span* msgid;    /* RFC5424 only, else NULL */
    const fg_span* msg;
    const fg_span* full_msg; /* on error rows of LTSV: off = byte offset of the failing part */
    const fg_span* sd;       /* {first entry, entry count} ; count 0 => Record.sd = None (always for RFC3164) */
    /* side table of LTSV / GELF, and of the RFC5424 wide rows */
    const fg_span* entry_name;  /* [n_entries] */
    const uint64_t* entry_val;  /* string: off | len<<32 ; bool/i64/u64/f64: the 8 value bytes ; header: #pairs */
    const uint8_t* entry_meta;  /* FG_EM_* */
    const int32_t* line_offsets; /* fg_split_decode only: [n+1] line starts into the stream (each line still
                                    carries its "\n" / "\r\n" terminator); NULL otherwise */
    /* RFC5424 (the columns ts .. sd above are NULL for this format) */
    const fg_row5424* rows5424; /* [n] */
    const uint64_t* entries8;   /* [n_entries8] */
    int32_t n_entries8;
    int32_t n_wide;             /* rows flagged FG_FLAG_WIDE */
    const fg_wide_row* wide_rows;
    const uint8_t* arena;       /* unescaped SD values (FG_E8_ARENA records, FG_EM_ARENA spans); RFC3164: re-joined messages (FG_FLAG_MSG_ARENA) */
    int64_t arena_bytes;
    /* timings of the call, milliseconds */
    float kernel_ms; /* sum of parse-kernel time (CUDA events on the launch stream) */
    float total_ms;  /* H2D + kernels + D2H wall time */
} fg_batch_out;

typedef struct fg_ctx fg_ctx;

/* 0 on success; negative FG_E_* otherwise.  Never throws, never aborts. */
#define FG_OK 0
#define FG_E_ARG (-1)
#define FG_E_CUDA (-2)
#define FG_E_CAPACITY (-3)
#define FG_E_NO_DEVICE (-4)

/* XDecoder::new(&Config) */
int fg_create(const fg_config* cfg, fg_ctx** out);
void fg_destroy(fg_ctx* ctx);
const char* fg_last_error(const fg_ctx* ctx); /* human-readable detail of the last negative return */

/* Pinned host arenas a batching splitter fills directly (no staging copy).
 * Any host pointer is accepted by fg_decode_batch; pinned ones go at PCIe rate. */
int fg_host_alloc(fg_ctx* ctx, size_t bytes, void** out);
void fg_host_free(fg_ctx* ctx, void* p);

/* RFC3164 environment after construction: the year (0 = follow the clock) and an explicit zone table.
 * Zone z is `names[z]` with spans [first[z], first[z+1]): span j holds UTC offset span_offset[j] (seconds east) from the UTC
 * second span_start_utc[j] on; the start of a zone's first span is ignored (it reaches back for ever).  A local time is
 * resolved as time-tz's assume_timezone does it (rfc3164_decoder.rs:202): the offset in force at that local time; a local
 * time that occurs twice takes the earlier offset, one that a forward jump skips the offset before the jump. */
int fg_set_rfc3164_year(fg_ctx* ctx, int32_t year);
int fg_set_tz_table(fg_ctx* ctx, int32_t n_zones, const char* const* names, const int32_t* first, const int64_t* span_start_utc,
                    const int32_t* span_offset);
/* Host-side queries of the zone database a context would load from `tzdir` (NULL as in fg_config); no device involved.
 * fg_tz_lookup: 1 = `name` is a zone (its UTC offset at local second `local` is stored), 0 = not a zone, <0 = no database. */
int fg_tz_lookup(const char* tzdir, const char* name, int64_t local, int32_t* offset);
int32_t fg_tz_count(const char* tzdir);

/* Decoder::decode for n lines.  offsets has n+1 monotone entries, offsets[0] >= 0;
 * line i is bytes[offsets[i] .. offsets[i+1]) and must be valid UTF-8 without the
 * line terminator (what LineSplitter hands to decode, line_splitter.rs:17-50). */
int fg_decode_batch(fg_ctx* ctx, fg_format fmt, const uint8_t* bytes, const int32_t* offsets, int32_t n,
                    fg_batch_out* out);

/* Framing + decoding in one call (SURVEY.md §8(f) N1): `stream` is a raw byte stream as LineSplitter::run reads it
 * (splitter/line_splitter.rs:17-25).  The device finds the '\n' terminators (BufRead::lines: the '\n' and one
 * preceding '\r' are dropped, an unterminated last line is still a line), validates every line as UTF-8 (an invalid
 * line gets status fg_error_string() == "Invalid UTF-8 input" and is not decoded) and decodes the rest.
 * Spans index `stream`; out->line_offsets locates the lines. */
int fg_split_decode(fg_ctx* ctx, fg_format fmt, const uint8_t* stream, int64_t nbytes, fg_batch_out* out);
/* The same with the framing of input.framing (mod.rs: "line" | "nul"): FG_FRAME_NUL is NulSplitter::run
 * (splitter/nul_splitter.rs:18-40): records end at a NUL byte, which is dropped (`BufRead::split(0)`), nothing else is
 * stripped, an unterminated last record is still a record, invalid UTF-8 => "Invalid UTF-8 input". */
typedef enum fg_framing { FG_FRAME_LINE = 0, FG_FRAME_NUL = 1 } fg_framing;
int fg_split_decode_framed(fg_ctx* ctx, fg_format fmt, fg_framing framing, const uint8_t* stream, int64_t nbytes, fg_batch_out* out);

/* Device-resident variant used for roofline measurement: fg_upload stages a
 * batch in HBM once; fg_parse_resident runs only the parse kernel(s) over it
 * and reports the CUDA-event time; fg_download fetches the result of the last
 * resident parse. */
int fg_upload(fg_ctx* ctx, const uint8_t* bytes, const int32_t* offsets, int32_t n);
int fg_parse_resident(fg_ctx* ctx, fg_format fmt, float* kernel_ms);
int fg_parse_resident_n(fg_ctx* ctx, fg_format fmt, int32_t k, float* total_ms); /* k passes, one host sync */
int fg_download(fg_ctx* ctx, fg_format fmt, fg_batch_out* out);
int fg_flush_l2(fg_ctx* ctx); /* writes a >L2-sized scratch buffer */

/* ---- decode + encode fused on the device (SURVEY.md 8(f) N2) ------------------------------------------------------
 * The reference calls Encoder::encode right after Decoder::decode for every record (splitter/line_splitter.rs:50-52).
 * For output.format = "gelf" with input.format = "rfc5424" (the default pair), "rfc3164", "ltsv" or "gelf" (a GELF
 * relay) both stages run on the GPU and only the encoded records come back:
 *     GelfEncoder::new(&Config)   encoder/gelf_encoder.rs:29-48   -> fg_set_gelf_extra (output.gelf_extra)
 *     Encoder::encode(Record)     encoder/gelf_encoder.rs:59-115, encoder/mod.rs:54-56 -> fg_decode_encode_gelf
 * Record i is bytes[offsets[i], offsets[i+1]) — exactly the Vec<u8> the reference's encode returns (serde_json 0.8
 * text: keys in byte order, later inserts replace earlier ones, no whitespace); a line the decoder rejects has
 * status[i] != 0 (fg_error_string) and an empty record.  An RFC3164 record has no application_name, process_id or sd_id
 * (the Record holds None for them; a gelf_extra of that key is still written), "level" only when the line has a <PRI>,
 * and "short_message" always (possibly ""), as rfc3164_decoder.rs builds it.  The year of a timestamp without one is
 * fixed at the start of each call (fg_set_rfc3164_year).  An LTSV record (ltsv_decoder.rs:87-221) has no
 * application_name, process_id or sd_id, "level" only when the line has a `level` part, "short_message" "-" without a
 * `message` part and "" for `message:`, and one "_" + name (+ the type's suffix, input.ltsv_suffixes) key per pair: a
 * later pair of the same key replaces an earlier one, and a schema-typed value is written as a JSON bool or number
 * (non-finite f64 -> null).  A GELF record (gelf_decoder.rs:34-125) has no application_name, process_id or sd_id,
 * "version":"1.1" whatever version the input named, "level" and "full_message" only when the object has them,
 * "short_message" "-" without one, "host" "unknown" for "", and one key per other member: "_" + its name, or the name
 * alone when it starts with '_' (a later member of the same key, in the order of the input's sorted keys, replaces an
 * earlier one); strings are written as serde_json escapes their unescaped text (`\/` -> `/`, `\u00e9` -> its UTF-8,
 * control bytes other than \b \f \n \r \t raw), numbers, booleans and null as JSON.  A record without "timestamp"
 * gets the wall clock read ONCE at the start of the call (fg_encoded_gelf_now), where the reference reads it per record
 * as it decodes: the two differ by at most the duration of the call.  LTSV or GELF input on a context not created for
 * that format (fg_config.input_format) -> FG_E_ARG. */
typedef struct fg_encoded_out {
    int32_t n;
    const uint8_t* bytes;     /* concatenated records, each framed by fg_set_output_framing */
    const int64_t* offsets;   /* [n+1] */
    const uint8_t* status;    /* [n] */
    float kernel_ms;          /* parse + encode kernels */
    float total_ms;
} fg_encoded_out;
int fg_set_gelf_extra(fg_ctx* ctx, int32_t n, const char* const* keys, const char* const* values);
/* output.framing: the Merger the Output applies to every encoded record before it writes it (src/flowgger/merger; picked
 * from output.framing in mod.rs:444-460; the caller resolves the reference's default and passes it here, as
 * fg_set_gelf_extra stands for GelfEncoder::new).  From the next fused call on, record i of fg_encoded_out is the bytes
 * the Output writes for it:
 *     FG_OUT_NONE    the record (the default; "noop" / "nop" / "none" / "capnp")
 *     FG_OUT_LINE    record "\n"                    (line_merger.rs:14)
 *     FG_OUT_NUL     record "\0"                    (nul_merger.rs:14)
 *     FG_OUT_SYSLEN  "{L + 1} " record "\n"          (syslen_merger.rs:15-28, L = the record's length in decimal)
 * A rejected record stays empty (no frame), so bytes[0, offsets[n]) is the whole output stream of the call, in input
 * order.  An unknown value -> FG_E_ARG, the context unchanged. */
typedef enum fg_out_framing { FG_OUT_NONE = 0, FG_OUT_LINE = 1, FG_OUT_NUL = 2, FG_OUT_SYSLEN = 3 } fg_out_framing;
int fg_set_output_framing(fg_ctx* ctx, fg_out_framing framing);
int fg_decode_encode_gelf(fg_ctx* ctx, fg_format fmt /* FG_FMT_RFC5424 | FG_FMT_RFC3164 | FG_FMT_LTSV | FG_FMT_GELF */,
                          const uint8_t* bytes, const int32_t* offsets, int32_t n, fg_encoded_out* out);
/* Raw stream -> framing (FG_FRAME_LINE | FG_FRAME_NUL, as fg_split_decode_framed) -> UTF-8 check -> RFC5424, RFC3164,
 * LTSV or GELF decode -> GelfEncoder::encode, all on the device; only the encoded records and the record extents come back.
 * Record i is out->bytes[out->offsets[i], out->offsets[i+1]); out->status[i] is 0, a decoder status, or the framing status
 * whose fg_error_string is "Invalid UTF-8 input" (empty record).  *line_offsets ([n+1], starts in `stream`, each record
 * still carrying its terminator, like fg_batch_out.line_offsets) stays valid until the next call on the context.
 * Errors: LTSV or GELF input on a context not created for that format, or an unknown framing -> FG_E_ARG;
 * nbytes > max_batch_bytes or more records than max_batch_lines -> FG_E_CAPACITY (the context stays usable). */
int fg_split_decode_encode_gelf(fg_ctx* ctx, fg_format fmt /* FG_FMT_RFC5424 | FG_FMT_RFC3164 | FG_FMT_LTSV | FG_FMT_GELF */, fg_framing framing,
                                const uint8_t* stream, int64_t nbytes, fg_encoded_out* out, const int32_t** line_offsets);
/* output.format = "ltsv" (encoder/ltsv_encoder.rs:10-123), the same four input formats:
 *     LTSVEncoder::new(&Config)   ltsv_encoder.rs:10-30   -> fg_set_ltsv_extra (output.ltsv_extra)
 *     Encoder::encode(Record)     ltsv_encoder.rs:66-123  -> fg_decode_encode_ltsv / fg_split_decode_encode_ltsv
 * Record i is the text LTSVEncoder::encode returns: `key:value` fields separated by '\t', in Record order with no sorting
 * and no de-duplication — every SD pair (its name without one leading '_': for LTSV input name + type suffix, for GELF
 * input the member's name without its '_'), the extras, host (as it is, "" included), time (Record.ts as Rust's
 * Display for f64: shortest round-trip digits, positional, no exponent: 1, 1000000000000000000000, 0.0000001, NaN, inf,
 * -0), then message, full_message, level, facility, appname, procid, msgid each only when the Record has it (RFC5424:
 * all; RFC3164: no appname / procid / msgid, level and facility only with a <PRI>; LTSV and GELF: no facility, appname,
 * procid or msgid).  In keys '\n' and '\t' become ' ' and ':' becomes '_'; in values '\t' and '\n' become ' '; nothing
 * else is escaped.  Typed values: true / false, f64 as above, decimal integers, null as "".  Everything else —
 * fg_encoded_out, statuses, empty rejected records, output.framing (fg_set_output_framing: the caller resolves the
 * reference's "line" default for ltsv), fg_encoded_ltsv_stops, fg_encoded_gelf_now, FG_E_CAPACITY, the input format
 * rule — is exactly as for the GELF twins above.
 * fg_set_ltsv_extra: the extras are written in byte order of their keys (a TOML table); a duplicate key or a NULL string
 * -> FG_E_ARG with the extras unchanged; n = 0 clears them. */
int fg_set_ltsv_extra(fg_ctx* ctx, int32_t n, const char* const* keys, const char* const* values);
int fg_decode_encode_ltsv(fg_ctx* ctx, fg_format fmt /* FG_FMT_RFC5424 | FG_FMT_RFC3164 | FG_FMT_LTSV | FG_FMT_GELF */,
                          const uint8_t* bytes, const int32_t* offsets, int32_t n, fg_encoded_out* out);
int fg_split_decode_encode_ltsv(fg_ctx* ctx, fg_format fmt /* FG_FMT_RFC5424 | FG_FMT_RFC3164 | FG_FMT_LTSV | FG_FMT_GELF */, fg_framing framing,
                                const uint8_t* stream, int64_t nbytes, fg_encoded_out* out, const int32_t** line_offsets);
/* output.format = "capnp" (encoder/capnp_encoder.rs:14-109, record.capnp), the same four input formats:
 *     CapnpEncoder::new(&Config)  capnp_encoder.rs:14-32   -> fg_set_capnp_extra (output.capnp_extra)
 *     Encoder::encode(Record)     capnp_encoder.rs:36-45   -> fg_decode_encode_capnp / fg_split_decode_encode_capnp
 * Record i is the message capnp::serialize::write_message writes for build_record's Record (capnp 0.14, a default
 * Builder): the segment table, then each segment's words.  Record = ts (f64), facility and severity (u8, 255 = None),
 * and the texts hostname, appname, procid, msgid, msg, fullMsg where the Record has them; of the FIRST SD element only,
 * sdId (RFC5424) and its pairs (key '_' + name, for LTSV input + the type suffix; string values as text, bool / f64 / i64
 * / u64 / null as the union's member); output.capnp_extra as the `extra` pairs, keys as given.  No byte is escaped; a
 * GELF string is its unescaped text.  A record up to 8 KiB or so is one segment; a longer one takes more, as capnp-rust's
 * HeapAllocator places them.  The reference writes no message holding a text of 2^29 - 1 bytes or more (capnp-rust
 * asserts): such a line fails the call with FG_E_ARG and a text naming the record, and no output is handed out.
 * Everything else — fg_encoded_out, statuses, empty rejected records, output.framing (the caller resolves the
 * reference's "noop" default for capnp: FG_OUT_NONE), fg_encoded_ltsv_stops, fg_encoded_gelf_now, FG_E_CAPACITY, the
 * input format rule — is exactly as for the GELF twins above.
 * fg_set_capnp_extra: the extras are written in byte order of their keys (a TOML table); a duplicate key, a NULL
 * string, a key or value of 2^29 - 1 bytes or more (no record could hold it) or more than 2^31 - 1 bytes of keys and
 * values in all -> FG_E_ARG with the extras unchanged; n = 0 clears them. */
int fg_set_capnp_extra(fg_ctx* ctx, int32_t n, const char* const* keys, const char* const* values);
int fg_decode_encode_capnp(fg_ctx* ctx, fg_format fmt /* FG_FMT_RFC5424 | FG_FMT_RFC3164 | FG_FMT_LTSV | FG_FMT_GELF */,
                           const uint8_t* bytes, const int32_t* offsets, int32_t n, fg_encoded_out* out);
int fg_split_decode_encode_capnp(fg_ctx* ctx, fg_format fmt /* FG_FMT_RFC5424 | FG_FMT_RFC3164 | FG_FMT_LTSV | FG_FMT_GELF */, fg_framing framing,
                                 const uint8_t* stream, int64_t nbytes, fg_encoded_out* out, const int32_t** line_offsets);
/* output.format = "passthrough" (encoder/passthrough_encoder.rs:10-46), the same four input formats:
 *     PassthroughEncoder::new(&Config)  passthrough_encoder.rs:11-14  -> fg_set_passthrough_prefix (the header)
 *     Encoder::encode(Record)           passthrough_encoder.rs:22-46  -> fg_decode_encode_passthrough /
 *                                                                         fg_split_decode_encode_passthrough
 * Record i is the header followed by Record.full_msg, byte for byte: for RFC5424 input the line after its BOM with
 * trailing Unicode White_Space removed, for RFC3164 the whole line (<PRI> included) trimmed the same way, for LTSV the
 * line as given, for GELF the unescaped full_message string ("" gives an accepted, empty record).  A GELF object without
 * full_message is the encoder's error: status FG_EP_NO_RAW = 128 (fg_error_string: "Cannot output empty raw message"), an
 * empty record and no frame, as a decoder error.  Everything else — fg_encoded_out, statuses, empty rejected records,
 * output.framing (the caller resolves the reference's default: "noop", FG_OUT_NONE, except "line" for output.type =
 * "debug"), fg_encoded_ltsv_stops, fg_encoded_gelf_now, FG_E_CAPACITY, the input format rule — is exactly as for the
 * GELF twins above.
 * fg_set_passthrough_prefix: the header of the following passthrough calls, written as given (any bytes, NUL and '\n'
 * included).  The reference formats output.syslog_prepend_timestamp per record (encoder/mod.rs:58-94); here the caller
 * formats it once per call (see fg_encoded_gelf_now for the same trade).  n = 0 clears it; NULL bytes with n > 0, or
 * n >= 2^31 -> FG_E_ARG with the header unchanged. */
int fg_set_passthrough_prefix(fg_ctx* ctx, const uint8_t* bytes, int64_t n);
int fg_decode_encode_passthrough(fg_ctx* ctx, fg_format fmt /* FG_FMT_RFC5424 | FG_FMT_RFC3164 | FG_FMT_LTSV | FG_FMT_GELF */,
                                 const uint8_t* bytes, const int32_t* offsets, int32_t n, fg_encoded_out* out);
int fg_split_decode_encode_passthrough(fg_ctx* ctx, fg_format fmt /* FG_FMT_RFC5424 | FG_FMT_RFC3164 | FG_FMT_LTSV | FG_FMT_GELF */,
                                       fg_framing framing, const uint8_t* stream, int64_t nbytes, fg_encoded_out* out,
                                       const int32_t** line_offsets);
/* The one side effect of LTSVDecoder::decode, println!("Missing value for name '{}'") for every tab-separated part
 * without ':' that the decode loop reached (ltsv_decoder.rs:99), for the records of the last fused call on an LTSV
 * context.  *stop ([out->n], valid until the next call on the context): -1 when record i printed nothing; else the offset,
 * relative to the record's start (offsets[i], or *line_offsets[i] in split mode), up to which its parts were read: the
 * failing part's offset on an error row, the record's length (without its terminator) + 1 otherwise.  Every part of the
 * record that starts before that offset and holds no ':' prints one line, in order.  A record that is not UTF-8 has -1.
 * Returns FG_E_ARG when the last fused call was not on LTSV input or failed. */
int fg_encoded_ltsv_stops(const fg_ctx* ctx, const int32_t** stop);
/* Record.ts of every record without "timestamp" in the last fused call on GELF input: CLOCK_REALTIME at the start of
 * that call, as secs + nanos / 1e9 (utils/mod.rs:16-21).  Returns FG_E_ARG when the last fused call was not on GELF
 * input or failed.
 * The passthrough header (fg_set_passthrough_prefix) makes the same trade: the reference formats
 * output.syslog_prepend_timestamp from OffsetDateTime::now_utc() per record, the device writes one header per call.  The
 * two differ only for the records the reference would have encoded after the clock crossed a tick of the format's
 * finest field (a second, a minute, ...) during the call. */
int fg_encoded_gelf_now(const fg_ctx* ctx, double* now);

/* the reference's Err(&'static str) for a row status (0 -> NULL).  fg_error_count: one past the largest status a decoder
 * or the framing gives; an encoder's status lies above every one of them (FG_EP_NO_RAW = 128, the passthrough encoder's
 * "Cannot output empty raw message"). */
const char* fg_error_string(fg_format fmt, uint32_t status);
uint32_t fg_error_count(void);

/* build/launch facts for tests and bench */
const char* fg_build_info(void);          /* arch, compiler, kernel list */
int64_t fg_kernel_launches(const fg_ctx* ctx); /* parse kernels launched by this ctx so far */
float fg_last_split_ms(const fg_ctx* ctx);     /* device time of the framing + UTF-8 kernels of the last fg_split_decode
                                                  (or fg_split_decode_framed / fg_split_decode_encode_gelf) */
float fg_last_dominant_kernel_ms(const fg_ctx* ctx); /* CUDA-event time of the dominant kernel alone (RFC5424: parse5424_kernel)
                                                        inside the last fg_parse_resident step */

#ifdef __cplusplus
}
#endif
#endif /* FLOWGGER_CUDA_H */
