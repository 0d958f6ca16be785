// flowgger.hpp — C++ host-side mirror of the reference's decoder-facing interface,
// layered on the C ABI (include/flowgger_cuda.h).
//
// The reference is Rust; no Rust toolchain exists in the build environment, so
// the code a flowgger maintainer would write in `cuda_decoder` (rust/cuda_decoder,
// shipped as source) is mirrored here 1:1 in C++ and is what the tests drive:
//   Record / StructuredData / SDValue      <- src/flowgger/record.rs:4-82
//   Decoder::decode / clone_boxed          <- src/flowgger/decoder/mod.rs:23-46
//   RFC5424Decoder / LTSVDecoder / GelfDecoder / RFC3164Decoder::new(&Config)
//                                          <- decoder/rfc5424_decoder.rs:12, ltsv_decoder.rs:24, gelf_decoder.rs:16, rfc3164_decoder.rs:14
//   BatchingLineSplitter::run              <- splitter/line_splitter.rs:10-54 (batched)
// All parsing happens in the CUDA kernels; this layer only packs lines, calls
// fg_decode_batch and materialises owned Records from the columnar spans.
#pragma once
#include <cstdint>
#include <functional>
#include <iosfwd>
#include <map>
#include <memory>
#include <mutex>
#include <optional>
#include <string>
#include <string_view>
#include <utility>
#include <vector>

#include "flowgger_cuda.h"

namespace flowgger {

// record.rs:4-11
struct SDValue {
    enum Kind : uint8_t { String = 0, Bool = 1, F64 = 2, I64 = 3, U64 = 4, Null = 5 } kind = Null;
    std::string s;
    union {
        bool b;
        double f;
        int64_t i;
        uint64_t u;
    };
    SDValue() : u(0) {}
};

// record.rs:24-27
struct StructuredData {
    std::optional<std::string> sd_id;
    std::vector<std::pair<std::string, SDValue>> pairs;
};

// record.rs:71-82
struct Record {
    double ts = 0.0;
    std::string hostname;
    std::optional<uint8_t> facility;
    std::optional<uint8_t> severity;
    std::optional<std::string> appname;
    std::optional<std::string> procid;
    std::optional<std::string> msgid;
    std::optional<std::string> msg;
    std::optional<std::string> full_msg;
    std::optional<std::vector<StructuredData>> sd;
};

// Result<Record, &'static str>
struct DecodeResult {
    const char* err = nullptr;  // nullptr = Ok
    Record record;
    bool ok() const { return err == nullptr; }
};

// input.ltsv_schema / input.ltsv_suffixes (ltsv_decoder.rs:24-83); type names are case-insensitive
struct LtsvConfig {
    bool has_schema = false;
    std::vector<std::pair<std::string, std::string>> schema;    // key -> "string"|"bool"|"f64"|"i64"|"u64"
    std::vector<std::pair<std::string, std::string>> suffixes;  // type -> suffix
};

struct DeviceOptions {
    int device = 0;
    int64_t max_batch_bytes = 0;
    int32_t max_batch_lines = 0;
    int32_t chunk_lines = 0;
    // input.format = "rfc3164": the year `OffsetDateTime::now_utc().year()` stands for (0 = follow the clock,
    // rfc3164_decoder.rs:175) and the TZif directory behind time_tz::timezones::get_by_name ("" = $TZDIR / system)
    int32_t rfc3164_year = 0;
    std::string tzdir;
};

// One GPU decoding context of a fixed format.  Single caller at a time (see mutex()).
class CudaFusedEncoder;

class CudaBatchDecoder {
   public:
    CudaBatchDecoder(fg_format fmt, const LtsvConfig& ltsv = {}, const DeviceOptions& opt = {});
    ~CudaBatchDecoder();
    CudaBatchDecoder(const CudaBatchDecoder&) = delete;
    CudaBatchDecoder& operator=(const CudaBatchDecoder&) = delete;

    fg_format format() const { return fmt_; }
    fg_ctx* ctx() const { return ctx_; }
    // serialises the callers that share this context (decoder clones): hold it from decode_batch until the last materialize
    std::mutex& mutex() { return mu_; }
    int64_t capacity_bytes() const { return opt_.max_batch_bytes; }
    int32_t capacity_lines() const { return opt_.max_batch_lines; }
    // a second context of the same format / LTSV configuration with another capacity (a single line larger than a batch)
    std::unique_ptr<CudaBatchDecoder> make_sized(int64_t max_batch_bytes, int32_t max_batch_lines) const;
    // packs nothing: bytes/offsets as in fg_decode_batch.  Throws std::runtime_error on a CUDA/argument failure.
    void decode_batch(const uint8_t* bytes, const int32_t* offsets, int32_t n, fg_batch_out* out);
    // Owned Record (or the reference's error string) of line i of a decoded batch.
    // `side_effects`, if given, receives the println! lines of ltsv_decoder.rs:99.
    DecodeResult materialize(const fg_batch_out& out, const uint8_t* bytes, const int32_t* offsets, int32_t i,
                             std::vector<std::string>* side_effects = nullptr) const;
    // same, for a line whose extent [line_lo, line_hi) is given explicitly (split mode: terminator already removed)
    DecodeResult materialize_line(const fg_batch_out& out, const uint8_t* bytes, int32_t line_lo, int32_t line_hi, int32_t i,
                                  std::vector<std::string>* side_effects = nullptr) const;
    // framing + UTF-8 validation + decode of a raw byte stream on the device (fg_split_decode)
    void split_decode(const uint8_t* stream, int64_t nbytes, fg_batch_out* out, fg_framing framing = FG_FRAME_LINE);
    // the same, but false (nothing decoded) when the stream does not fit the context: more bytes or more records
    bool try_split_decode(const uint8_t* stream, int64_t nbytes, fg_batch_out* out, fg_framing framing);
    // decode + GelfEncoder::encode fused on the device (fg_decode_encode_gelf); `extra` = output.gelf_extra, `out_framing`
    // = output.framing (fg_set_output_framing)
    void decode_encode_gelf(const uint8_t* bytes, const int32_t* offsets, int32_t n,
                            const std::vector<std::pair<std::string, std::string>>& extra, fg_encoded_out* out,
                            fg_out_framing out_framing = FG_OUT_NONE);
    // framing + decode + GelfEncoder::encode fused on the device (fg_split_decode_encode_gelf); false as try_split_decode
    bool try_split_decode_encode_gelf(const uint8_t* stream, int64_t nbytes, fg_framing framing,
                                      const std::vector<std::pair<std::string, std::string>>& extra, fg_encoded_out* out,
                                      const int32_t** line_offsets, fg_out_framing out_framing = FG_OUT_NONE);
    // the two calls above for either fused encoder (output format, extras and output.framing from `enc`)
    void decode_encode(const CudaFusedEncoder& enc, const uint8_t* bytes, const int32_t* offsets, int32_t n, fg_encoded_out* out);
    bool try_split_decode_encode(const CudaFusedEncoder& enc, const uint8_t* stream, int64_t nbytes, fg_framing framing,
                                 fg_encoded_out* out, const int32_t** line_offsets);
    // after one of the fused calls on an LTSV context: where each record's "Missing value" lines stop
    // (fg_encoded_ltsv_stops, for ltsv_missing_values); nullptr for other formats
    const int32_t* encoded_ltsv_stops() const;

   private:
    void set_encoder(const CudaFusedEncoder& enc);
    fg_format fmt_;
    fg_ctx* ctx_ = nullptr;
    std::mutex mu_;
    std::vector<std::pair<std::string, std::string>> extra_set_[3];  // per CudaFusedEncoder::Output
    bool extra_valid_[3] = {false, false, false};
    LtsvConfig ltsv_;
    DeviceOptions opt_;
    std::string suffix_[5];
    bool has_suffix_[5] = {false, false, false, false, false};
};

// decoder/mod.rs:44-46 + :23-36
class Decoder {
   public:
    virtual ~Decoder() = default;
    virtual DecodeResult decode(std::string_view line) const = 0;
    virtual std::unique_ptr<Decoder> clone_boxed() const = 0;
    virtual std::shared_ptr<CudaBatchDecoder> batch() const = 0;
};

// Drop-in decoders: `decode(line)` is a batch of one through the same kernels.
class CudaDecoder : public Decoder {
   public:
    CudaDecoder(fg_format fmt, const LtsvConfig& ltsv = {}, const DeviceOptions& opt = {});
    DecodeResult decode(std::string_view line) const override;
    std::unique_ptr<Decoder> clone_boxed() const override;
    std::shared_ptr<CudaBatchDecoder> batch() const override { return impl_; }

   private:
    explicit CudaDecoder(std::shared_ptr<CudaBatchDecoder> impl) : impl_(std::move(impl)) {}
    std::shared_ptr<CudaBatchDecoder> impl_;
};
struct RFC5424Decoder : CudaDecoder {
    explicit RFC5424Decoder(const DeviceOptions& opt = {}) : CudaDecoder(FG_FMT_RFC5424, {}, opt) {}
};
struct LTSVDecoder : CudaDecoder {
    explicit LTSVDecoder(const LtsvConfig& cfg = {}, const DeviceOptions& opt = {}) : CudaDecoder(FG_FMT_LTSV, cfg, opt) {}
};
struct GelfDecoder : CudaDecoder {
    explicit GelfDecoder(const DeviceOptions& opt = {}) : CudaDecoder(FG_FMT_GELF, {}, opt) {}
};
// decoder/rfc3164_decoder.rs:10-17 (the Config is unused there as well)
struct RFC3164Decoder : CudaDecoder {
    explicit RFC3164Decoder(const DeviceOptions& opt = {}) : CudaDecoder(FG_FMT_RFC3164, {}, opt) {}
};

// encoder/mod.rs:54-56 (interface only: encoders are out of scope, SURVEY.md §8(f) N2)
class Encoder {
   public:
    virtual ~Encoder() = default;
    virtual bool encode(Record&& record, std::vector<uint8_t>& out, const char** err) const = 0;
};

// encoder/gelf_encoder.rs:10-48: output.format = "gelf".  The encoder runs FUSED with the decoder on the GPU
// (fg_decode_encode_gelf) for the input formats fuses_with() accepts: the batching splitters and RecordBatcher recognise
// this type and never materialise Records for them (for LTSV they print the decoder's "Missing value" lines from
// fg_encoded_ltsv_stops; GELF prints nothing, and its records without "timestamp" carry the wall clock of the call,
// fg_encoded_gelf_now).  `out_framing` = output.framing, applied on the device as well (fg_set_output_framing): with a
// framing other than FG_OUT_NONE the fused paths send ONE buffer per device call, the framed records of the whole
// batch, exactly what the Output writes, and the Output gets no merger.
// A fused encoder, and which output format it writes: what RecordEmitter, RecordBatcher and the batching splitters need
// to run it on the device (CudaBatchDecoder::decode_encode / try_split_decode_encode).
class CudaFusedEncoder : public Encoder {
   public:
    enum class Output { Gelf, Ltsv, Capnp, Passthrough };
    // the decoders whose device-resident results the fused encoders read
    static bool fuses_with(fg_format fmt) {
        return fmt == FG_FMT_RFC5424 || fmt == FG_FMT_RFC3164 || fmt == FG_FMT_LTSV || fmt == FG_FMT_GELF;
    }
    // a lone host-side Record cannot be encoded: there is no CPU encoder behind this interface
    bool encode(Record&&, std::vector<uint8_t>&, const char** err) const override {
        static const char* const kWhat[] = {"GelfEncoder runs fused with the decoder on the GPU (use BatchingLineSplitter)",
                                            "LTSVEncoder runs fused with the decoder on the GPU (use BatchingLineSplitter)",
                                            "CapnpEncoder runs fused with the decoder on the GPU (use BatchingLineSplitter)",
                                            "PassthroughEncoder runs fused with the decoder on the GPU (use BatchingLineSplitter)"};
        if (err) *err = kWhat[(int)output_];
        return false;
    }
    Output output() const { return output_; }
    // output.gelf_extra, output.ltsv_extra or output.capnp_extra
    const std::vector<std::pair<std::string, std::string>>& extra() const { return extra_; }
    fg_out_framing out_framing() const { return out_framing_; }
    // Output::Passthrough: the header of the records of one device call, asked once per call (none: no header)
    const std::function<std::string()>& header() const { return header_; }

   protected:
    CudaFusedEncoder(Output output, std::vector<std::pair<std::string, std::string>> extra, fg_out_framing out_framing,
                     std::function<std::string()> header = {})
        : output_(output), extra_(std::move(extra)), out_framing_(out_framing), header_(std::move(header)) {}

   private:
    Output output_;
    std::vector<std::pair<std::string, std::string>> extra_;
    fg_out_framing out_framing_;
    std::function<std::string()> header_;
};

class CudaGelfEncoder : public CudaFusedEncoder {
   public:
    explicit CudaGelfEncoder(std::vector<std::pair<std::string, std::string>> extra = {}, fg_out_framing out_framing = FG_OUT_NONE)
        : CudaFusedEncoder(Output::Gelf, std::move(extra), out_framing) {}
};

// encoder/ltsv_encoder.rs:10-30: output.format = "ltsv", fused with the decoder on the GPU as CudaGelfEncoder is
// (fg_decode_encode_ltsv).  `extra` = output.ltsv_extra (written in byte order of its keys), `out_framing` =
// output.framing (the caller resolves the reference's "line" default for ltsv, mod.rs:444-460).
class CudaLtsvEncoder : public CudaFusedEncoder {
   public:
    explicit CudaLtsvEncoder(std::vector<std::pair<std::string, std::string>> extra = {}, fg_out_framing out_framing = FG_OUT_NONE)
        : CudaFusedEncoder(Output::Ltsv, std::move(extra), out_framing) {}
};

// encoder/capnp_encoder.rs:14-45: output.format = "capnp", fused with the decoder on the GPU as CudaGelfEncoder is
// (fg_decode_encode_capnp).  `extra` = output.capnp_extra (written in byte order of its keys), `out_framing` =
// output.framing: FG_OUT_NONE is the reference's "noop" default for capnp (mod.rs:444-460).
class CudaCapnpEncoder : public CudaFusedEncoder {
   public:
    explicit CudaCapnpEncoder(std::vector<std::pair<std::string, std::string>> extra = {}, fg_out_framing out_framing = FG_OUT_NONE)
        : CudaFusedEncoder(Output::Capnp, std::move(extra), out_framing) {}
};

// encoder/passthrough_encoder.rs:10-46: output.format = "passthrough", fused with the decoder on the GPU as
// CudaGelfEncoder is (fg_decode_encode_passthrough): each record is the header + Record.full_msg.  `header` =
// output.syslog_prepend_timestamp formatted for the current time, called once per device call before it runs (none: no
// header); `out_framing` = output.framing, resolved by the caller (the reference's default: "noop", FG_OUT_NONE, and
// "line" for output.type = "debug", mod.rs:444-451).  A GELF record without full_message gets the encoder's error
// (FG_EP_NO_RAW) on stderr, as a decoder error.
class CudaPassthroughEncoder : public CudaFusedEncoder {
   public:
    explicit CudaPassthroughEncoder(std::function<std::string()> header = {}, fg_out_framing out_framing = FG_OUT_NONE)
        : CudaFusedEncoder(Output::Passthrough, {}, out_framing, std::move(header)) {}
};

// What RecordBatcher and the batching splitters do with each record of a batch decoded on the device, one record at a
// time in stream order, as the reference's per-record call sites do: LTSV's "Missing value" lines on stdout
// (ltsv_decoder.rs:99), then the encoded record to `tx`, or "{err}: [{line.trim()}]" / "Invalid UTF-8 input" on stderr.
// The caller gives record i's extent [lo, hi) in its bytes, without the terminator.
class RecordEmitter {
   public:
    RecordEmitter(const Encoder& encoder, std::function<void(std::vector<uint8_t>&&)> tx, std::ostream& err_out,
                  std::ostream& std_out, bool quiet_blank);
    // the encoder when it runs fused with the decoder of `gpu` (CudaFusedEncoder::fuses_with), else nullptr
    const CudaFusedEncoder* fused_with(const CudaBatchDecoder& gpu) const;
    // record i of a fused call on a decoder of format `fmt`; `stops` = CudaBatchDecoder::encoded_ltsv_stops()
    void emit(fg_format fmt, const fg_encoded_out& eo, const int32_t* stops, const uint8_t* bytes, int32_t i, int32_t lo,
              int32_t hi);
    // record i of a batch `gpu` decoded: materialised and encoded on the host
    void emit(const CudaBatchDecoder& gpu, const fg_batch_out& out, const uint8_t* bytes, int32_t i, int32_t lo, int32_t hi);
    // after the records of a fused call: with output.framing, the framed records of the whole call in one `tx`
    void end_batch(const fg_encoded_out& eo);
    // "Invalid UTF-8 input" on stderr (line_splitter.rs:22-25, nul_splitter.rs:25)
    void invalid_utf8();

   private:
    void reject(fg_format fmt, uint32_t status, const char* err, const uint8_t* bytes, int32_t lo, int32_t hi);
    const Encoder& encoder_;
    const CudaFusedEncoder* fused_;
    std::function<void(std::vector<uint8_t>&&)> tx_;
    std::ostream& err_;
    std::ostream& out_;
    bool quiet_blank_;  // nothing on stderr for a blank rejected record (the NUL splitter)
    std::vector<std::string> fx_;  // side effects of the record in hand
};

// The batching twin of the reference's per-record call sites (`decode -> encode -> tx.send`, or print
// "{err}: [{line.trim()}]" to stderr): line_splitter.rs:50, nul_splitter.rs:57, syslen_splitter.rs:65,
// input/udp_input.rs:139, input/redis_input.rs:159, input/file/worker.rs:116.  A caller frames its records as the old
// code did and push()es each one; the batcher accumulates up to Limits, decodes the batch on the GPU in one call and then,
// in the original order, encodes + sends every Record or prints the identical stderr line.  With a CudaGelfEncoder and a
// decoder it fuses with (CudaGelfEncoder::fuses_with) the two stages run fused on the device (fg_decode_encode_gelf).
class RecordBatcher {
   public:
    struct Limits {
        int32_t max_lines = 1 << 16;
        int64_t max_bytes = 16 << 20;
    };
    RecordBatcher(const Decoder& decoder, const Encoder& encoder, std::function<void(std::vector<uint8_t>&&)> tx,
                  std::ostream& err_out, std::ostream& std_out, Limits lim, bool quiet_blank = false);
    void push(std::string_view record);        // one framed record (valid UTF-8)
    void invalid_utf8() { ++invalid_before_.back(); }  // a record that failed the UTF-8 check: reported in stream order
    void flush() { flush_on(gpu_.get()); }     // call on max_lines / max_bytes (automatic), input-idle timeout and EOF

   private:
    void flush_on(CudaBatchDecoder* gpu);
    std::shared_ptr<CudaBatchDecoder> gpu_;
    RecordEmitter emit_;
    int64_t max_bytes_;
    int32_t max_lines_;
    std::vector<uint8_t> arena_;
    std::vector<int32_t> offsets_{0};
    std::vector<int32_t> invalid_before_{0};  // "Invalid UTF-8 input" events, kept in stream order relative to the records
};

// Batched twin of LineSplitter::run (splitter/line_splitter.rs:10-54).  It reads raw blocks of up to Limits::max_bytes
// (at most the context's max_batch_bytes), cuts each after its last "\n" and carries the tail into the next block.  The
// device frames the block like BufRead::lines (strip "\n" and one "\r"), checks UTF-8 (invalid => "Invalid UTF-8 input"
// on stderr, line skipped) and decodes it (fg_split_decode_framed); with a CudaGelfEncoder and a decoder it fuses with
// (CudaGelfEncoder::fuses_with) it also encodes (fg_split_decode_encode_gelf).  A block that frames into more lines than the context holds is decoded in two
// halves cut at a "\n" near its middle; a line longer than max_batch_bytes gets a context of its own (make_sized).
class BatchingLineSplitter {
   public:
    struct Limits {
        int32_t max_lines = 1 << 16;
        int64_t max_bytes = 16 << 20;
    };
    BatchingLineSplitter() = default;
    explicit BatchingLineSplitter(Limits l) : lim_(l) {}
    // tx: receives each encoded record; err_out/std_out: the reference's stderr/stdout text
    void run(std::istream& in, const std::function<void(std::vector<uint8_t>&&)>& tx, const Decoder& decoder,
             const Encoder& encoder, std::ostream& err_out, std::ostream& std_out) const;

   private:
    Limits lim_;
};
// Batched twins of NulSplitter::run (splitter/nul_splitter.rs:10-47: raw blocks framed on the device, as
// BatchingLineSplitter with NUL delimiters) and SyslenSplitter::run (syslen_splitter.rs:10-57: framed on the host, fed
// to a RecordBatcher)
class BatchingNulSplitter {
   public:
    BatchingNulSplitter() = default;
    explicit BatchingNulSplitter(BatchingLineSplitter::Limits l) : lim_(l) {}
    void run(std::istream& in, const std::function<void(std::vector<uint8_t>&&)>& tx, const Decoder& decoder,
             const Encoder& encoder, std::ostream& err_out, std::ostream& std_out) const;

   private:
    BatchingLineSplitter::Limits lim_;
};
class BatchingSyslenSplitter {
   public:
    BatchingSyslenSplitter() = default;
    explicit BatchingSyslenSplitter(BatchingLineSplitter::Limits l) : lim_(l) {}
    void run(std::istream& in, const std::function<void(std::vector<uint8_t>&&)>& tx, const Decoder& decoder,
             const Encoder& encoder, std::ostream& err_out, std::ostream& std_out) const;

   private:
    BatchingLineSplitter::Limits lim_;
};

// §8(e): lines are independent, so a batch shards across GPUs by contiguous line ranges balanced by BYTES
// (binary search on the offsets prefix); no collective, results concatenate in shard order.
// bounds has G+1 entries: shard g covers lines [bounds[g], bounds[g+1]).
void shard_by_bytes(const int32_t* offsets, int32_t n, int G, int32_t* bounds);

// One CudaBatchDecoder per device + one host thread per device.
class MultiGpuBatchDecoder {
   public:
    MultiGpuBatchDecoder(fg_format fmt, const std::vector<int>& devices, const LtsvConfig& ltsv = {},
                         const DeviceOptions& per_device = {});
    int shards() const { return (int)dec_.size(); }
    struct Shard {
        int32_t line0 = 0, n = 0;     // lines [line0, line0+n) of the batch
        int64_t byte_base = 0;        // spans of this shard are relative to bytes + byte_base
        fg_batch_out out{};
        std::vector<int32_t> offsets; // rebased offsets handed to the device
    };
    // decodes the batch on all devices concurrently; shard g's result stays valid until the next call
    const std::vector<Shard>& decode_batch(const uint8_t* bytes, const int32_t* offsets, int32_t n);
    DecodeResult materialize(int32_t line, const uint8_t* bytes, std::vector<std::string>* side_effects = nullptr) const;
    CudaBatchDecoder& device(int g) { return *dec_[(size_t)g]; }

   private:
    std::vector<std::unique_ptr<CudaBatchDecoder>> dec_;
    std::vector<Shard> shards_;
};

// Owned Record (or the reference's error string) of line i = bytes[line_lo, line_hi) of a decoded batch; `suffix` = the
// five LTSV type suffixes (may be null for other formats).  Pure function of the result arrays: no device, no context.
DecodeResult materialize_record(fg_format fmt, const std::string* suffix, const fg_batch_out& out, const uint8_t* bytes,
                                int32_t line_lo, int32_t line_hi, int32_t i, std::vector<std::string>* side_effects);
// The println! of ltsv_decoder.rs:99 for the LTSV record bytes[lo, hi): "Missing value for name '{part}'" for every
// tab-separated part without ':' that starts before `stop` (absolute; hi + 1 = every part), appended to `out` in order
void ltsv_missing_values(const uint8_t* bytes, int32_t lo, int32_t hi, int32_t stop, std::vector<std::string>& out);
uint32_t row_meta(const fg_batch_out& out, int32_t i);

// helpers shared with tests
bool is_valid_utf8(const uint8_t* p, size_t n);
std::string_view rust_trim(std::string_view s);
void dump_result(const DecodeResult& r, bool ts_is_now, const std::vector<std::string>& side_effects, std::string& out);

}  // namespace flowgger
