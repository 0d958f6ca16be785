// fg_status.h — per-line status codes shared by the kernels and the C ABI.
// Each code maps 1:1 onto one `&'static str` the reference decoders return
// (file:line cited in fg_abi.cu's string table).  Order inside a format follows
// the reference's evaluation order (SURVEY.md §8(a) error-code table).
#pragma once
#include <stdint.h>

enum FgStatus : uint32_t {
    FG_ST_OK = 0,
    // RFC5424 (decoder/rfc5424_decoder.rs)
    FG_E5_BOM = 1,
    FG_E5_PRI_BRACKETS = 2,
    FG_E5_INVALID_PRI = 3,
    FG_E5_MISSING_VERSION = 4,
    FG_E5_UNSUPPORTED_VERSION = 5,
    FG_E5_MISSING_TS = 6,
    FG_E5_BAD_TS = 7,
    FG_E5_MISSING_HOST = 8,
    FG_E5_MISSING_APP = 9,
    FG_E5_MISSING_PROCID = 10,
    FG_E5_MISSING_MSGID = 11,
    FG_E5_MISSING_DATA = 12,
    FG_E5_MISSING_MSG = 13,
    FG_E5_MALFORMED = 14,
    FG_E5_MISSING_SD = 15,
    FG_E5_SD_FORMAT = 16,
    FG_E5_SD_NO_END = 17,
    FG_E5_MISSING_PRI_VERSION = 18,  // unreachable in the reference (splitn always yields one item)
    FG_E5_EMPTY_PRI = 19,            // unreachable
    FG_E5_MISSING_SD_ID = 20,        // unreachable
    // LTSV (decoder/ltsv_decoder.rs)
    FG_EL_TS = 32,
    FG_EL_SEV = 33,
    FG_EL_SEV_HIGH = 34,
    FG_EL_BOOL = 35,
    FG_EL_F64 = 36,
    FG_EL_I64 = 37,
    FG_EL_U64 = 38,
    FG_EL_MISSING_TS = 39,
    FG_EL_MISSING_HOST = 40,
    // GELF (decoder/gelf_decoder.rs)
    FG_EG_JSON = 64,
    FG_EG_EMPTY = 65,
    FG_EG_TS = 66,
    FG_EG_HOST = 67,
    FG_EG_SHORT = 68,
    FG_EG_FULL = 69,
    FG_EG_VERSION_T = 70,
    FG_EG_VERSION = 71,
    FG_EG_SEV = 72,
    FG_EG_SEV_HIGH = 73,
    FG_EG_SD_TYPE = 74,
    FG_EG_MISSING_HOST = 75,
    // framing (splitter/line_splitter.rs:22-25): not a decoder error; the line is skipped with this stderr text
    FG_ES_INVALID_UTF8 = 76,
    // RFC3164 (decoder/rfc3164_decoder.rs); the error of the LAST form tried is the one returned (:40-47)
    FG_E3_PRI_MALFORMED = 80,  // '<' without '>'
    FG_E3_PRI_INVALID = 81,
    FG_E3_CUSTOM = 82,         // fewer than three ": " pieces
    FG_E3_TIME_FORMAT = 83,    // fewer than three date tokens
    FG_E3_WITH_YEAR = 84,      // three date tokens that do not parse without a year
    FG_E3_DATE = 85,
    FG_E3_PANIC = 86,          // `_log_tokens[0]` on an empty Vec (:64): the reference thread panics
    FG_ST_COUNT = 87,          // decoder and framing statuses are 1 .. FG_ST_COUNT - 1 (fg_error_count)
    // Encoder statuses lie above every decoder status: an encoder's Err for a Record the decoder accepted.
    // passthrough encoder (encoder/passthrough_encoder.rs:44): a Record without full_msg (only GELF input has one)
    FG_EP_NO_RAW = 128
};
