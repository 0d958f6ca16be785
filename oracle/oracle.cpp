// oracle/oracle.cpp — TEST INFRASTRUCTURE, NOT PRODUCT CODE (see oracle.hpp).
//
// Line-by-line CPU restatement of the reference decoders.  Every function
// cites the reference lines it follows (paths relative to
// flowgger src/flowgger/).  Like the reference it builds an owned
// Record (one heap string per field) so that it is also a fair CPU baseline.
#include "oracle.hpp"

#include <charconv>
#include <cinttypes>
#include <clocale>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <locale.h>
#include <memory>

namespace fgo {

// ---------------------------------------------------------------------------
// Rust std primitives (SURVEY.md Appendix B)
// ---------------------------------------------------------------------------

// char::is_whitespace (Unicode White_Space) decoded from UTF-8 at the FRONT of
// s; returns the encoded length (0 = not whitespace).
static size_t ws_len_front(std::string_view s) {
    if (s.empty()) return 0;
    unsigned char c0 = (unsigned char)s[0];
    if ((c0 >= 0x09 && c0 <= 0x0D) || c0 == 0x20) return 1;
    if (c0 == 0xC2 && s.size() >= 2) {
        unsigned char c1 = (unsigned char)s[1];
        return (c1 == 0x85 || c1 == 0xA0) ? 2 : 0;  // U+0085, U+00A0
    }
    if (s.size() >= 3) {
        unsigned char c1 = (unsigned char)s[1], c2 = (unsigned char)s[2];
        if (c0 == 0xE1) return (c1 == 0x9A && c2 == 0x80) ? 3 : 0;  // U+1680
        if (c0 == 0xE2) {
            if (c1 == 0x80 && ((c2 >= 0x80 && c2 <= 0x8A) || c2 == 0xA8 || c2 == 0xA9 || c2 == 0xAF))
                return 3;  // U+2000-200A, U+2028, U+2029, U+202F
            if (c1 == 0x81 && c2 == 0x9F) return 3;  // U+205F
            return 0;
        }
        if (c0 == 0xE3) return (c1 == 0x80 && c2 == 0x80) ? 3 : 0;  // U+3000
    }
    return 0;
}

// same, for the character ENDING at the back of s
static size_t ws_len_back(std::string_view s) {
    size_t n = s.size();
    if (n == 0) return 0;
    unsigned char l = (unsigned char)s[n - 1];
    if (l < 0x80) return ((l >= 0x09 && l <= 0x0D) || l == 0x20) ? 1 : 0;
    // multi-byte: walk back to the lead byte (input is valid UTF-8)
    size_t k = 1;
    while (k < 4 && k < n && (((unsigned char)s[n - k]) & 0xC0) == 0x80) ++k;
    std::string_view ch = s.substr(n - k, k);
    size_t w = ws_len_front(ch);
    return (w == k) ? k : 0;
}

std::string_view rust_trim_end(std::string_view s) {
    for (;;) {
        size_t w = ws_len_back(s);
        if (!w) return s;
        s.remove_suffix(w);
    }
}
static std::string_view rust_trim_start(std::string_view s) {
    for (;;) {
        size_t w = ws_len_front(s);
        if (!w) return s;
        s.remove_prefix(w);
    }
}
std::string_view rust_trim(std::string_view s) { return rust_trim_start(rust_trim_end(s)); }

// core::num from_str_radix(10) for unsigned types: [+]digit+, overflow = Err
bool rust_parse_u64(std::string_view s, uint64_t& out) {
    if (s.empty()) return false;
    size_t i = 0;
    if (s[0] == '+') {
        i = 1;
    }
    if (i >= s.size()) return false;  // "" or lone "+"  (a lone "-" is an invalid digit below)
    uint64_t v = 0;
    for (; i < s.size(); ++i) {
        unsigned d = (unsigned char)s[i] - '0';
        if (d > 9) return false;
        if (v > (UINT64_MAX - d) / 10) return false;
        v = v * 10 + d;
    }
    out = v;
    return true;
}
bool rust_parse_u8(std::string_view s, uint8_t& out) {
    if (s.empty()) return false;
    size_t i = (s[0] == '+') ? 1 : 0;
    if (i >= s.size()) return false;
    unsigned v = 0;
    for (; i < s.size(); ++i) {
        unsigned d = (unsigned char)s[i] - '0';
        if (d > 9) return false;
        v = v * 10 + d;
        if (v > 255) return false;
    }
    out = (uint8_t)v;
    return true;
}
bool rust_parse_i64(std::string_view s, int64_t& out) {
    if (s.empty()) return false;
    size_t i = 0;
    bool neg = false;
    if (s[0] == '+') i = 1;
    else if (s[0] == '-') { i = 1; neg = true; }
    if (i >= s.size()) return false;
    uint64_t lim = neg ? (uint64_t)1 << 63 : (uint64_t)INT64_MAX;
    uint64_t v = 0;
    for (; i < s.size(); ++i) {
        unsigned d = (unsigned char)s[i] - '0';
        if (d > 9) return false;
        if (v > (lim - d) / 10) return false;
        v = v * 10 + d;
    }
    out = neg ? (int64_t)(0 - v) : (int64_t)v;
    return true;
}

static bool ieq(std::string_view a, const char* b) {
    size_t n = strlen(b);
    if (a.size() != n) return false;
    for (size_t i = 0; i < n; ++i) {
        char c = a[i];
        if (c >= 'A' && c <= 'Z') c = (char)(c + 32);
        if (c != b[i]) return false;
    }
    return true;
}

// f64::from_str (core::num::dec2flt): [+-](inf|infinity|nan | digits[.digits][e[+-]digits])
// correctly rounded, overflow -> inf, underflow -> 0.  Grammar enforced here,
// the correctly rounded conversion is delegated to glibc strtod in the C locale.
bool rust_parse_f64(std::string_view s, double& out) {
    if (s.empty()) return false;
    size_t i = 0;
    bool neg = false;
    if (s[0] == '+' || s[0] == '-') { neg = s[0] == '-'; i = 1; }
    std::string_view r = s.substr(i);
    if (r.empty()) return false;
    if (ieq(r, "inf") || ieq(r, "infinity")) { out = neg ? -INFINITY : INFINITY; return true; }
    if (ieq(r, "nan")) {
        uint64_t bits = 0x7ff8000000000000ULL | (neg ? 0x8000000000000000ULL : 0);
        memcpy(&out, &bits, 8);
        return true;
    }
    size_t p = 0, nint = 0, nfrac = 0;
    while (p < r.size() && r[p] >= '0' && r[p] <= '9') { ++p; ++nint; }
    if (p < r.size() && r[p] == '.') {
        ++p;
        while (p < r.size() && r[p] >= '0' && r[p] <= '9') { ++p; ++nfrac; }
    }
    if (nint + nfrac == 0) return false;
    std::string norm;
    norm.reserve(r.size() + 4);
    if (nint == 0) norm.push_back('0');
    norm.append(r.substr(0, p));
    if (nfrac == 0 && !norm.empty() && norm.back() == '.') norm.push_back('0');
    if (p < r.size()) {
        if (r[p] != 'e' && r[p] != 'E') return false;
        ++p;
        size_t es = p;
        if (p < r.size() && (r[p] == '+' || r[p] == '-')) ++p;
        size_t ed = p;
        while (p < r.size() && r[p] >= '0' && r[p] <= '9') ++p;
        if (p == ed || p != r.size()) return false;
        norm.push_back('e');
        norm.append(r.substr(es, p - es));
    }
    static locale_t cloc = newlocale(LC_ALL_MASK, "C", (locale_t)0);
    char* end = nullptr;
    double v = strtod_l(norm.c_str(), &end, cloc);
    out = neg ? -v : v;
    return true;
}

static bool rust_parse_bool(std::string_view s, bool& out) {
    if (s == "true") { out = true; return true; }
    if (s == "false") { out = false; return true; }
    return false;
}

// ---------------------------------------------------------------------------
// `time` 0.3 restatement: calendar, Rfc3339, the English format description
// (time crate is not vendored: algorithm restated from its published source;
//  call sites rfc5424_decoder.rs:95, ltsv_decoder.rs:225,249-250)
// ---------------------------------------------------------------------------

static bool is_leap(int64_t y) { return (y % 4 == 0 && y % 100 != 0) || y % 400 == 0; }
static int days_in_month(int64_t y, int m) {
    static const int d[12] = {31, 28, 31, 30, 31, 30, 31, 31, 30, 31, 30, 31};
    return (m == 2 && is_leap(y)) ? 29 : d[m - 1];
}
// proleptic Gregorian days since 1970-01-01
static int64_t days_from_civil(int64_t y, int m, int d) {
    y -= m <= 2;
    int64_t era = (y >= 0 ? y : y - 399) / 400;
    int64_t yoe = y - era * 400;
    int64_t doy = (153 * (m + (m > 2 ? -3 : 9)) + 2) / 5 + d - 1;
    int64_t doe = yoe * 365 + yoe / 4 - yoe / 100 + doy;
    return era * 146097 + doe - 719468;
}

struct DateTimeParts {
    int64_t year = 0;
    int month = 0, day = 0, hour = 0, minute = 0, second = 0;
    uint32_t nanos = 0;
    int offset_seconds = 0;
};

// utils/mod.rs:24-28: `tsd.unix_timestamp_nanos() as f64 / 1e9`
// (i128 -> f64 is one IEEE RNE rounding, the division a second one)
static double nanos_to_ts(__int128 nanos) {
    double f = (double)nanos;  // libgcc __floattidf: round-to-nearest-even
    return f / 1e9;
}

static bool finish_datetime(const DateTimeParts& p, bool leap_second_input, double& out) {
    // Month::from_number, Date::from_calendar_date, Time::from_hms_nano
    if (p.month < 1 || p.month > 12) return false;
    if (p.year < -9999 || p.year > 9999) return false;
    if (p.day < 1 || p.day > days_in_month(p.year, p.month)) return false;
    if (p.hour > 23 || p.minute > 59 || p.second > 59) return false;
    __int128 local = (__int128)days_from_civil(p.year, p.month, p.day) * 86400 +
                     p.hour * 3600 + p.minute * 60 + p.second;
    __int128 utc = local - p.offset_seconds;
    if (leap_second_input) {
        // OffsetDateTime::is_valid_leap_second_stand_in: 23:59:59.999999999 UTC
        // on the last day of a month.
        if (p.nanos != 999999999u) return false;
        int64_t u = (int64_t)utc;
        int64_t days = u >= 0 ? u / 86400 : -((-u + 86399) / 86400);
        int64_t sod = u - days * 86400;
        if (sod != 86399) return false;
        // civil_from_days
        int64_t z = days + 719468;
        int64_t era = (z >= 0 ? z : z - 146096) / 146097;
        int64_t doe = z - era * 146097;
        int64_t yoe = (doe - doe / 1460 + doe / 36524 - doe / 146096) / 365;
        int64_t y = yoe + era * 400;
        int64_t doy = doe - (365 * yoe + yoe / 4 - yoe / 100);
        int64_t mp = (5 * doy + 2) / 153;
        int d = (int)(doy - (153 * mp + 2) / 5 + 1);
        int m = (int)(mp < 10 ? mp + 3 : mp - 9);
        y += m <= 2;
        if (d != days_in_month(y, m)) return false;
    }
    out = nanos_to_ts(utc * 1000000000 + p.nanos);
    return true;
}

static bool two_digits(std::string_view s, size_t& i, int& out) {
    if (i + 2 > s.size()) return false;
    unsigned a = (unsigned char)s[i] - '0', b = (unsigned char)s[i + 1] - '0';
    if (a > 9 || b > 9) return false;
    out = (int)(a * 10 + b);
    i += 2;
    return true;
}
static bool lit(std::string_view s, size_t& i, char c) {
    if (i < s.size() && s[i] == c) { ++i; return true; }
    return false;
}
static bool lit_ic(std::string_view s, size_t& i, char upper) {
    if (i < s.size() && (s[i] == upper || s[i] == (char)(upper + 32))) { ++i; return true; }
    return false;
}
// any_digit+ with the `time` truncation rule (digits past the 9th are consumed and dropped)
static bool subsecond(std::string_view s, size_t& i, uint32_t& nanos) {
    if (i >= s.size() || s[i] < '0' || s[i] > '9') return false;
    uint32_t value = (uint32_t)(s[i] - '0') * 100000000u;
    ++i;
    uint32_t mult = 10000000u;
    while (i < s.size() && s[i] >= '0' && s[i] <= '9') {
        value += (uint32_t)(s[i] - '0') * mult;
        mult /= 10;
        ++i;
    }
    nanos = value;
    return true;
}
// UtcOffset::from_hms range (time >= 0.3.21: |h| <= 25, |m| <= 59)
static bool offset_ok(int h, int m) { return h <= 25 && m <= 59; }

// time::OffsetDateTime::parse(s, &Rfc3339)  (time/src/parsing/parsable.rs, impl for Rfc3339)
bool rfc3339_to_unix(std::string_view s, double& out) {
    size_t i = 0;
    DateTimeParts p;
    if (s.size() < 4) return false;
    int64_t y = 0;
    for (int k = 0; k < 4; ++k) {
        unsigned d = (unsigned char)s[k] - '0';
        if (d > 9) return false;
        y = y * 10 + d;
    }
    p.year = y;
    i = 4;
    if (!lit(s, i, '-') || !two_digits(s, i, p.month) || !lit(s, i, '-') || !two_digits(s, i, p.day)) return false;
    if (!lit_ic(s, i, 'T')) return false;
    if (!two_digits(s, i, p.hour) || !lit(s, i, ':') || !two_digits(s, i, p.minute) || !lit(s, i, ':') ||
        !two_digits(s, i, p.second))
        return false;
    if (lit(s, i, '.')) {
        if (!subsecond(s, i, p.nanos)) return false;
    }
    if (lit_ic(s, i, 'Z')) {
        p.offset_seconds = 0;
    } else {
        if (i >= s.size() || (s[i] != '+' && s[i] != '-')) return false;
        bool neg = s[i] == '-';
        ++i;
        int oh = 0, om = 0;
        if (!two_digits(s, i, oh) || !lit(s, i, ':') || !two_digits(s, i, om)) return false;
        if (!offset_ok(oh, om)) return false;
        p.offset_seconds = (oh * 3600 + om * 60) * (neg ? -1 : 1);
    }
    if (i != s.size()) return false;  // UnexpectedTrailingCharacters
    bool leap = false;
    if (p.second == 60) {
        p.second = 59;
        p.nanos = 999999999u;
        leap = true;
    }
    return finish_datetime(p, leap, out);
}

// ltsv_decoder.rs:236-254:
//   "[day padding:none]/[month repr:short]/[year]:[hour]:[minute]:[second](.[subsecond]) [offset_hour sign:mandatory][offset_minute]"
bool english_to_unix(std::string_view s, bool with_subsecond, double& out) {
    static const char* MON[12] = {"Jan", "Feb", "Mar", "Apr", "May", "Jun", "Jul", "Aug", "Sep", "Oct", "Nov", "Dec"};
    size_t i = 0;
    DateTimeParts p;
    // [day padding:none]: 1..2 digits greedy, NonZero
    if (i >= s.size() || s[i] < '0' || s[i] > '9') return false;
    p.day = s[i++] - '0';
    if (i < s.size() && s[i] >= '0' && s[i] <= '9') p.day = p.day * 10 + (s[i++] - '0');
    if (p.day == 0) return false;
    if (!lit(s, i, '/')) return false;
    if (i + 3 > s.size()) return false;
    p.month = 0;
    for (int m = 0; m < 12; ++m)
        if (s.compare(i, 3, MON[m]) == 0) { p.month = m + 1; break; }
    if (!p.month) return false;
    i += 3;
    if (!lit(s, i, '/')) return false;
    // [year]: optional sign, exactly 4 digits
    bool yneg = false;
    if (i < s.size() && (s[i] == '+' || s[i] == '-')) { yneg = s[i] == '-'; ++i; }
    if (i + 4 > s.size()) return false;
    int64_t y = 0;
    for (int k = 0; k < 4; ++k) {
        unsigned d = (unsigned char)s[i + k] - '0';
        if (d > 9) return false;
        y = y * 10 + d;
    }
    i += 4;
    p.year = yneg ? -y : y;
    if (!lit(s, i, ':') || !two_digits(s, i, p.hour) || !lit(s, i, ':') || !two_digits(s, i, p.minute) ||
        !lit(s, i, ':') || !two_digits(s, i, p.second))
        return false;
    if (with_subsecond) {
        if (!lit(s, i, '.') || !subsecond(s, i, p.nanos)) return false;
    }
    if (!lit(s, i, ' ')) return false;
    if (i >= s.size() || (s[i] != '+' && s[i] != '-')) return false;  // sign:mandatory
    bool neg = s[i] == '-';
    ++i;
    int oh = 0, om = 0;
    if (!two_digits(s, i, oh) || !two_digits(s, i, om)) return false;
    if (!offset_ok(oh, om)) return false;
    p.offset_seconds = (oh * 3600 + om * 60) * (neg ? -1 : 1);
    if (i != s.size()) return false;
    return finish_datetime(p, false, out);  // second == 60 rejected (no leap seconds for custom formats)
}

// ---------------------------------------------------------------------------
// RFC5424  (decoder/rfc5424_decoder.rs)
// ---------------------------------------------------------------------------

static const char* const E5_BOM = "Unsupported BOM";
static const char* const E5_PRI_BRACKETS = "The priority should be inside brackets";
static const char* const E5_INVALID_PRI = "Invalid priority";
static const char* const E5_MISSING_VERSION = "Missing version";
static const char* const E5_UNSUPPORTED_VERSION = "Unsupported version";
static const char* const E5_MISSING_TS = "Missing timestamp";
static const char* const E5_BAD_TS = "Unable to parse the date from RFC3339 to Unix time in RFC5424 decoder";
static const char* const E5_MISSING_HOST = "Missing hostname";
static const char* const E5_MISSING_APP = "Missing application name";
static const char* const E5_MISSING_PROCID = "Missing process id";
static const char* const E5_MISSING_MSGID = "Missing message id";
static const char* const E5_MISSING_DATA = "Missing message data";
static const char* const E5_MISSING_MSG = "Missing log message";
static const char* const E5_MALFORMED = "Malformated RFC5424 message";
static const char* const E5_MISSING_SD = "Missing structured data";
static const char* const E5_SD_FORMAT = "Format error in the structured data";
static const char* const E5_SD_NO_END = "Missing ] after structured data";

// rfc5424_decoder.rs:105-125
static std::string unescape_sd_value(std::string_view value) {
    std::string res;
    bool esc = false;
    for (char c : value) {
        if (!esc) {
            if (c == '\\') esc = true;
            else res.push_back(c);
        } else {
            if (c == '"' || c == '\\' || c == ']') {
                res.push_back(c);
            } else {
                res.push_back('\\');
                res.push_back(c);
            }
            esc = false;
        }
    }
    return res;
}

// rfc5424_decoder.rs:163-172
static std::optional<std::string> parse_msg(std::string_view line, size_t offset) {
    if (offset > line.size()) return std::nullopt;
    std::string_view m = rust_trim(line.substr(offset));
    if (m.empty()) return std::nullopt;
    return std::string(m);
}

// rfc5424_decoder.rs:174-242.  Returns error or fills sd / leftover / after-offset.
static const char* parse_sd_data(std::string_view line, size_t offset, StructuredData& sd_res,
                                 std::string_view& leftover, size_t& after) {
    std::string_view rest = line.substr(offset);
    size_t sp = rest.find(' ');
    if (sp == std::string_view::npos) return E5_MISSING_SD;  // :177
    std::string_view sd_id = rest.substr(0, sp);
    std::string_view sd = rest.substr(sp + 1);
    bool in_name = false, in_value = false, esc = false, have_name = false;
    size_t name_start = 0, value_start = 0;
    std::string_view name;
    bool found_end = false;
    size_t after_sd = 0;
    sd_res.sd_id = std::string(sd_id);
    // byte-wise evaluation is equivalent to char-wise: every deciding char is ASCII
    for (size_t i = 0; i < sd.size(); ++i) {
        unsigned char c = (unsigned char)sd[i];
        bool is_sd_name = (c >= 33 && c <= 126) && c != 34 && c != 61 && c != 93;  // :188-192
        if (c == ' ' && !esc && !in_name && !have_name) {  // :194
        } else if (c == ']' && !esc && !in_name && !have_name) {  // :197
            after_sd = i + 1;
            found_end = true;
            break;
        } else if (!esc && is_sd_name && !in_name && !have_name) {  // :201
            in_name = true;
            name_start = i;
        } else if (is_sd_name && in_name && !have_name) {  // :205
        } else if (c == '=' && !esc && in_name) {  // :208
            name = sd.substr(name_start, i - name_start);
            have_name = true;
            in_name = false;
        } else if (c == '"' && !esc && have_name && !in_value) {  // :212
            in_value = true;
            value_start = i + 1;
        } else if (c == '\\' && !esc && in_value) {  // :216
            esc = true;
        } else if (c == '"' && !esc && in_value) {  // :217
            in_value = false;
            SDValue v;
            v.tag = SDTag::String;
            v.s = unescape_sd_value(sd.substr(value_start, i - value_start));
            sd_res.pairs.emplace_back("_" + std::string(name), std::move(v));
            have_name = false;
        } else if (in_value) {  // :231
            esc = false;
        } else if (c == '"' && !esc && !in_name && !have_name) {  // :232
        } else {
            return E5_SD_FORMAT;  // :235
        }
    }
    if (!found_end) return E5_SD_NO_END;  // :239
    leftover = sd;
    after = after_sd;
    return nullptr;
}

// rfc5424_decoder.rs:127-161
static const char* parse_data(std::string_view line, std::vector<StructuredData>& sd_vec,
                              std::optional<std::string>& msg) {
    if (line.empty()) return E5_MISSING_MSG;  // :129
    char c0 = line[0];
    if (c0 == '-') {
        msg = parse_msg(line, 1);
        return nullptr;
    }
    if (c0 != '[') return E5_MALFORMED;  // :159
    std::string_view leftover = line;
    size_t offset = 0;
    for (;;) {
        StructuredData sd;
        std::string_view nl;
        size_t noff = 0;
        if (const char* e = parse_sd_data(leftover, offset + 1, sd, nl, noff)) return e;
        leftover = nl;
        offset = noff;
        sd_vec.push_back(std::move(sd));
        if (offset >= leftover.size()) return E5_MISSING_MSG;  // :148
        char c = leftover[offset];
        if (c == '[') continue;
        if (c == ' ') {
            msg = parse_msg(leftover, offset);
            return nullptr;
        }
        return E5_MALFORMED;  // :154
    }
}

// rfc5424_decoder.rs:18-49
Decoded rfc5424_decode(std::string_view line) {
    Decoded d;
    // BOM::parse :63-71
    if (line.size() >= 3 && (unsigned char)line[0] == 0xEF && (unsigned char)line[1] == 0xBB &&
        (unsigned char)line[2] == 0xBF) {
        line.remove_prefix(3);
    } else if (!line.empty() && line[0] == '<') {
    } else {
        d.err = E5_BOM;
        return d;
    }
    // splitn(7, ' ')
    std::string_view parts[7];
    int nparts = 0;
    {
        std::string_view rest = line;
        while (nparts < 6) {
            size_t sp = rest.find(' ');
            if (sp == std::string_view::npos) break;
            parts[nparts++] = rest.substr(0, sp);
            rest = rest.substr(sp + 1);
        }
        parts[nparts++] = rest;
    }
    // parse_pri_version :74-92
    {
        std::string_view pv = parts[0];
        if (pv.empty() || pv[0] != '<') { d.err = E5_PRI_BRACKETS; return d; }
        std::string_view r = pv.substr(1);
        size_t gt = r.find('>');
        std::string_view pri_s = gt == std::string_view::npos ? r : r.substr(0, gt);
        uint8_t pri = 0;
        if (!rust_parse_u8(pri_s, pri)) { d.err = E5_INVALID_PRI; return d; }
        if (gt == std::string_view::npos) { d.err = E5_MISSING_VERSION; return d; }
        if (r.substr(gt + 1) != "1") { d.err = E5_UNSUPPORTED_VERSION; return d; }
        d.rec.facility = (uint8_t)(pri >> 3);
        d.rec.severity = (uint8_t)(pri & 7);
    }
    if (nparts < 2) { d.err = E5_MISSING_TS; return d; }
    if (!rfc3339_to_unix(parts[1], d.rec.ts)) { d.err = E5_BAD_TS; return d; }
    if (nparts < 3) { d.err = E5_MISSING_HOST; return d; }
    if (nparts < 4) { d.err = E5_MISSING_APP; return d; }
    if (nparts < 5) { d.err = E5_MISSING_PROCID; return d; }
    if (nparts < 6) { d.err = E5_MISSING_MSGID; return d; }
    if (nparts < 7) { d.err = E5_MISSING_DATA; return d; }
    std::vector<StructuredData> sd_vec;
    std::optional<std::string> msg;
    if (const char* e = parse_data(parts[6], sd_vec, msg)) { d.err = e; return d; }
    d.rec.hostname = std::string(parts[2]);
    d.rec.appname = std::string(parts[3]);
    d.rec.procid = std::string(parts[4]);
    d.rec.msgid = std::string(parts[5]);
    if (!sd_vec.empty()) d.rec.sd = std::move(sd_vec);
    d.rec.msg = std::move(msg);
    d.rec.full_msg = std::string(rust_trim_end(line));
    return d;
}

// ---------------------------------------------------------------------------
// LTSV  (decoder/ltsv_decoder.rs)
// ---------------------------------------------------------------------------

static const char* const EL_TS = "Unable to parse the English to Unix timestamp in LTSV decoder";
static const char* const EL_SEV = "Invalid severity level";
static const char* const EL_SEV_HIGH = "Severity level should be <= 7";
static const char* const EL_BOOL = "Type error; boolean was expected";
static const char* const EL_F64 = "Type error; f64 was expected";
static const char* const EL_I64 = "Type error; i64 was expected";
static const char* const EL_U64 = "Type error; u64 was expected";
static const char* const EL_MISSING_TS = "Missing timestamp";
static const char* const EL_MISSING_HOST = "Missing hostname";

// ltsv_decoder.rs:263-267
static bool ltsv_parse_ts(std::string_view s, double& out) {
    if (rust_parse_f64(s, out)) return true;        // unix_strtime_to_unix :256-261
    if (rfc3339_to_unix(s, out)) return true;       // :224-229
    if (english_to_unix(s, false, out)) return true;  // :231-234
    return english_to_unix(s, true, out);
}

static bool ends_with(std::string_view s, std::string_view suf) {
    return s.size() >= suf.size() && s.substr(s.size() - suf.size()) == suf;
}

Decoded ltsv_decode(const LtsvConfig& cfg, std::string_view line) {
    Decoded d;
    StructuredData sd;
    std::optional<double> ts;
    std::optional<std::string> hostname, msg;
    std::optional<uint8_t> severity;
    size_t pos = 0;
    for (;;) {  // line.split('\t') :94
        size_t tab = line.find('\t', pos);
        std::string_view part = tab == std::string_view::npos ? line.substr(pos) : line.substr(pos, tab - pos);
        size_t colon = part.find(':');  // splitn(2, ':') :95
        if (colon == std::string_view::npos) {
            d.stdout_lines.push_back("Missing value for name '" + std::string(part) + "'");  // :99
        } else {
            std::string_view name = part.substr(0, colon), value = part.substr(colon + 1);
            if (name == "time") {  // :104-111
                std::string_view ts_s = value;
                if (!value.empty() && value.front() == '[' && value.back() == ']') {
                    // value "[" alone would make &value[1..0] panic in Rust; starts_with && ends_with
                    // on a 1-byte "[" is false for ends_with(']'), so len >= 2 here.
                    ts_s = value.substr(1, value.size() - 2);
                }
                double t;
                if (!ltsv_parse_ts(ts_s, t)) { d.err = EL_TS; return d; }
                ts = t;
            } else if (name == "host") {
                hostname = std::string(value);
            } else if (name == "message") {
                msg = std::string(value);
            } else if (name == "level") {  // :114-121
                uint8_t sev;
                if (!rust_parse_u8(value, sev)) { d.err = EL_SEV; return d; }
                if (sev > 7) { d.err = EL_SEV_HIGH; return d; }
                severity = sev;
            } else {  // :122-199
                SDValue v;
                std::string final_name = "_" + std::string(name);
                SDType t = SDType::String;
                if (cfg.has_schema) {
                    auto it = cfg.schema.find(std::string(name));
                    if (it != cfg.schema.end()) t = it->second;
                }
                const std::optional<std::string>* suf = nullptr;
                switch (t) {
                    case SDType::String:
                        v.tag = SDTag::String;
                        v.s = std::string(value);
                        break;
                    case SDType::Bool:
                        suf = &cfg.suffix_bool;
                        v.tag = SDTag::Bool;
                        if (!rust_parse_bool(value, v.b)) { d.err = EL_BOOL; return d; }
                        break;
                    case SDType::F64:
                        suf = &cfg.suffix_f64;
                        v.tag = SDTag::F64;
                        if (!rust_parse_f64(value, v.f)) { d.err = EL_F64; return d; }
                        break;
                    case SDType::I64:
                        suf = &cfg.suffix_i64;
                        v.tag = SDTag::I64;
                        if (!rust_parse_i64(value, v.i)) { d.err = EL_I64; return d; }
                        break;
                    case SDType::U64:
                        suf = &cfg.suffix_u64;
                        v.tag = SDTag::U64;
                        if (!rust_parse_u64(value, v.u)) { d.err = EL_U64; return d; }
                        break;
                }
                if (suf && suf->has_value() && !ends_with(name, **suf)) final_name += **suf;
                sd.pairs.emplace_back(std::move(final_name), std::move(v));
            }
        }
        if (tab == std::string_view::npos) break;
        pos = tab + 1;
    }
    if (!ts) { d.err = EL_MISSING_TS; return d; }          // :205
    if (!hostname) { d.err = EL_MISSING_HOST; return d; }  // :206
    d.rec.ts = *ts;
    d.rec.hostname = std::move(*hostname);
    d.rec.severity = severity;
    if (!sd.pairs.empty()) {
        std::vector<StructuredData> v;
        v.push_back(std::move(sd));
        d.rec.sd = std::move(v);
    }
    d.rec.msg = std::move(msg);
    d.rec.full_msg = std::string(line);
    return d;
}

// ---------------------------------------------------------------------------
// serde_json ~0.8 restatement (crate not vendored; algorithm restated from its
// published source: de.rs parse_value/parse_integer/parse_decimal/
// parse_exponent/visit_f64_from_parts, read.rs parse_str_bytes/parse_escape,
// value.rs Value + BTreeMap object).  Call sites gelf_decoder.rs:42-49.
// ---------------------------------------------------------------------------

struct JValue {
    enum T : uint8_t { Null, Bool, I64, U64, F64, String, Array, Object } t = Null;
    bool b = false;
    int64_t i = 0;
    uint64_t u = 0;
    double f = 0;
    std::string s;
    std::vector<JValue> arr;
    std::map<std::string, JValue> obj;  // BTreeMap<String, Value>: byte-lexicographic, insert replaces
};

enum class JErr { None, Syntax, InvalidUnicodeCodePoint };

struct JParser {
    std::string_view in;
    size_t i = 0;
    int remaining_depth = 128;
    JErr err = JErr::None;

    bool fail(JErr e = JErr::Syntax) { if (err == JErr::None) err = e; return false; }
    int peek() const { return i < in.size() ? (unsigned char)in[i] : -1; }
    void ws() {
        while (i < in.size() && (in[i] == ' ' || in[i] == '\n' || in[i] == '\t' || in[i] == '\r')) ++i;
    }
    bool ident(const char* rest) {
        for (const char* p = rest; *p; ++p) {
            if (i >= in.size() || in[i] != *p) return fail();
            ++i;
        }
        return true;
    }
    static bool overflow_u64(uint64_t a, uint64_t b) {  // overflow!(a * 10 + b, u64::MAX)
        return a >= UINT64_MAX / 10 && (a > UINT64_MAX / 10 || b > UINT64_MAX % 10);
    }
    bool f64_from_parts(bool pos, uint64_t significand, int32_t exponent, JValue& out) {
        static double POW10[309];
        static bool init = false;
        if (!init) {
            // exact decimal literals 1e0..1e308, correctly rounded like rustc's table
            for (int k = 0; k <= 308; ++k) {
                char buf[16];
                snprintf(buf, sizeof buf, "1e%d", k);
                POW10[k] = strtod(buf, nullptr);
            }
            init = true;
        }
        double f = (double)significand;
        for (;;) {
            int64_t ae = exponent < 0 ? -(int64_t)exponent : exponent;
            if (ae <= 308) {
                double pw = POW10[ae];
                if (exponent >= 0) {
                    f *= pw;
                    if (std::isinf(f)) return fail();
                } else {
                    f /= pw;
                }
                break;
            }
            if (f == 0.0) break;
            if (exponent >= 0) return fail();
            f /= 1e308;
            exponent += 308;
        }
        out.t = JValue::F64;
        out.f = pos ? f : -f;
        return true;
    }
    bool parse_exponent(bool pos, uint64_t significand, int32_t starting_exp, JValue& out) {
        ++i;  // 'e'
        bool pos_exp = true;
        if (peek() == '+') ++i;
        else if (peek() == '-') { ++i; pos_exp = false; }
        int c = peek();
        if (c < '0' || c > '9') { if (c >= 0) ++i; return fail(); }
        ++i;
        int32_t exp = c - '0';
        while (peek() >= '0' && peek() <= '9') {
            int digit = peek() - '0';
            ++i;
            if (exp >= INT32_MAX / 10 && (exp > INT32_MAX / 10 || digit > INT32_MAX % 10)) {
                // parse_exponent_overflow
                if (significand != 0 && pos_exp) return fail();
                while (peek() >= '0' && peek() <= '9') ++i;
                out.t = JValue::F64;
                out.f = pos ? 0.0 : -0.0;
                return true;
            }
            exp = exp * 10 + digit;
        }
        int64_t fe = pos_exp ? (int64_t)starting_exp + exp : (int64_t)starting_exp - exp;  // saturating
        if (fe > INT32_MAX) fe = INT32_MAX;
        if (fe < INT32_MIN) fe = INT32_MIN;
        return f64_from_parts(pos, significand, (int32_t)fe, out);
    }
    bool parse_decimal(bool pos, uint64_t significand, int32_t exponent, JValue& out) {
        ++i;  // '.'
        bool at_least_one = false;
        while (peek() >= '0' && peek() <= '9') {
            uint64_t digit = (uint64_t)(peek() - '0');
            ++i;
            at_least_one = true;
            if (overflow_u64(significand, digit)) {
                while (peek() >= '0' && peek() <= '9') ++i;
                break;
            }
            significand = significand * 10 + digit;
            exponent -= 1;
        }
        if (!at_least_one) return fail();
        if (peek() == 'e' || peek() == 'E') return parse_exponent(pos, significand, exponent, out);
        return f64_from_parts(pos, significand, exponent, out);
    }
    bool parse_number(bool pos, uint64_t significand, JValue& out) {
        int c = peek();
        if (c == '.') return parse_decimal(pos, significand, 0, out);
        if (c == 'e' || c == 'E') return parse_exponent(pos, significand, 0, out);
        if (pos) {
            out.t = JValue::U64;
            out.u = significand;
        } else {
            int64_t neg = (int64_t)(0 - significand);  // (significand as i64).wrapping_neg()
            if (neg > 0) {
                out.t = JValue::F64;
                out.f = -(double)significand;
            } else if (neg < 0) {
                out.t = JValue::I64;
                out.i = neg;
            } else {
                out.t = JValue::U64;  // Value visitor: visit_i64(0) -> U64(0)
                out.u = 0;
            }
        }
        return true;
    }
    bool parse_long_integer(bool pos, uint64_t significand, int32_t exponent, JValue& out) {
        for (;;) {
            int c = peek();
            if (c >= '0' && c <= '9') { ++i; exponent += 1; }
            else if (c == '.') return parse_decimal(pos, significand, exponent, out);
            else if (c == 'e' || c == 'E') return parse_exponent(pos, significand, exponent, out);
            else return f64_from_parts(pos, significand, exponent, out);
        }
    }
    bool parse_integer(bool pos, JValue& out) {
        int c = peek();
        if (c < 0) return fail();
        ++i;
        if (c == '0') {
            if (peek() >= '0' && peek() <= '9') return fail();
            return parse_number(pos, 0, out);
        }
        if (c >= '1' && c <= '9') {
            uint64_t res = (uint64_t)(c - '0');
            for (;;) {
                int p = peek();
                if (p >= '0' && p <= '9') {
                    ++i;
                    uint64_t digit = (uint64_t)(p - '0');
                    if (overflow_u64(res, digit)) return parse_long_integer(pos, res, 1, out);
                    res = res * 10 + digit;
                } else {
                    return parse_number(pos, res, out);
                }
            }
        }
        return fail();
    }
    bool hex4(unsigned& n) {
        n = 0;
        for (int k = 0; k < 4; ++k) {
            if (i >= in.size()) return fail();
            unsigned char c = (unsigned char)in[i++];
            unsigned v;
            if (c >= '0' && c <= '9') v = c - '0';
            else if (c >= 'a' && c <= 'f') v = c - 'a' + 10;
            else if (c >= 'A' && c <= 'F') v = c - 'A' + 10;
            else return fail();
            n = n * 16 + v;
        }
        return true;
    }
    static void push_utf8(std::string& s, unsigned cp) {
        if (cp < 0x80) s.push_back((char)cp);
        else if (cp < 0x800) { s.push_back((char)(0xC0 | (cp >> 6))); s.push_back((char)(0x80 | (cp & 0x3F))); }
        else if (cp < 0x10000) {
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
    bool parse_str(std::string& out) {  // opening quote already consumed
        out.clear();
        for (;;) {
            if (i >= in.size()) return fail();  // EOFWhileParsingString
            unsigned char c = (unsigned char)in[i];
            if (c == '"') { ++i; return true; }
            if (c == '\\') {
                ++i;
                if (i >= in.size()) return fail();
                unsigned char e = (unsigned char)in[i++];
                switch (e) {
                    case '"': out.push_back('"'); break;
                    case '\\': out.push_back('\\'); break;
                    case '/': out.push_back('/'); break;
                    case 'b': out.push_back('\x08'); break;
                    case 'f': out.push_back('\x0c'); break;
                    case 'n': out.push_back('\n'); break;
                    case 'r': out.push_back('\r'); break;
                    case 't': out.push_back('\t'); break;
                    case 'u': {
                        unsigned n1;
                        if (!hex4(n1)) return false;
                        if (n1 >= 0xDC00 && n1 <= 0xDFFF) return fail();  // LoneLeadingSurrogateInHexEscape
                        if (n1 >= 0xD800 && n1 <= 0xDBFF) {
                            if (i + 2 > in.size()) return fail();
                            if (in[i] != '\\' || in[i + 1] != 'u') { i += 2; return fail(); }
                            i += 2;
                            unsigned n2;
                            if (!hex4(n2)) return false;
                            if (n2 < 0xDC00 || n2 > 0xDFFF) return fail();
                            unsigned n = (((n1 - 0xD800) << 10) | (n2 - 0xDC00)) + 0x10000;
                            push_utf8(out, n);
                        } else {
                            push_utf8(out, n1);
                        }
                        break;
                    }
                    default: return fail();  // InvalidEscape
                }
                continue;
            }
            if (c < 0x20) return fail(JErr::InvalidUnicodeCodePoint);  // raw control char in string
            out.push_back((char)c);
            ++i;
        }
    }
    bool parse_value(JValue& out) {
        ws();
        int c = peek();
        if (c < 0) return fail();  // EOFWhileParsingValue
        switch (c) {
            case 'n': ++i; if (!ident("ull")) return false; out.t = JValue::Null; return true;
            case 't': ++i; if (!ident("rue")) return false; out.t = JValue::Bool; out.b = true; return true;
            case 'f': ++i; if (!ident("alse")) return false; out.t = JValue::Bool; out.b = false; return true;
            case '-': ++i; return parse_integer(false, out);
            case '"': ++i; out.t = JValue::String; return parse_str(out.s);
            case '[': {
                if (--remaining_depth == 0) return fail();  // RecursionLimitExceeded
                ++i;
                out.t = JValue::Array;
                bool first = true;
                for (;;) {
                    ws();
                    int p = peek();
                    if (p < 0) return fail();
                    if (p == ']') { ++i; break; }
                    if (p == ',' && !first) ++i;
                    else if (first) first = false;
                    else return fail();
                    JValue v;
                    if (!parse_value(v)) return false;
                    out.arr.push_back(std::move(v));
                }
                ++remaining_depth;
                return true;
            }
            case '{': {
                if (--remaining_depth == 0) return fail();
                ++i;
                out.t = JValue::Object;
                bool first = true;
                for (;;) {
                    ws();
                    int p = peek();
                    if (p < 0) return fail();
                    if (p == '}') { ++i; break; }
                    if (p == ',' && !first) { ++i; ws(); }
                    else if (first) first = false;
                    else return fail();
                    if (peek() != '"') return fail();  // KeyMustBeAString / EOF
                    ++i;
                    std::string key;
                    if (!parse_str(key)) return false;
                    ws();
                    if (peek() != ':') return fail();
                    ++i;
                    JValue v;
                    if (!parse_value(v)) return false;
                    out.obj[std::move(key)] = std::move(v);  // BTreeMap::insert: last duplicate wins
                }
                ++remaining_depth;
                return true;
            }
            default:
                if (c >= '0' && c <= '9') return parse_integer(true, out);
                return fail();  // ExpectedSomeValue
        }
    }
    bool parse_document(JValue& out) {
        if (!parse_value(out)) return false;
        ws();
        if (i != in.size()) return fail();  // TrailingCharacters
        return true;
    }
};

// ---------------------------------------------------------------------------
// GELF  (decoder/gelf_decoder.rs)
// ---------------------------------------------------------------------------

static const char* const EG_JSON = "Invalid GELF input, unable to parse as a JSON object";
static const char* const EG_EMPTY = "Empty GELF input";
static const char* const EG_TS = "Invalid GELF timestamp";
static const char* const EG_HOST = "GELF host name must be a string";
static const char* const EG_SHORT = "GELF short message must be a string";
static const char* const EG_FULL = "GELF full message must be a string";
static const char* const EG_VERSION_T = "GELF version must be a string";
static const char* const EG_VERSION = "Unsupported GELF version";
static const char* const EG_SEV = "Invalid severity level";
static const char* const EG_SEV_HIGH = "Invalid severity level (too high)";
static const char* const EG_SD_TYPE = "Invalid value type in structured data";
static const char* const EG_MISSING_HOST = "Missing hostname";

Decoded gelf_decode(std::string_view line) {
    Decoded d;
    JValue root;
    {
        JParser p;
        p.in = line;
        if (!p.parse_document(root)) {
            if (p.err != JErr::InvalidUnicodeCodePoint) { d.err = EG_JSON; return d; }
            // gelf_decoder.rs:44-46: retry with every '\n' replaced by the two bytes `\n`
            std::string repl;
            repl.reserve(line.size() + 8);
            for (char c : line) {
                if (c == '\n') { repl.push_back('\\'); repl.push_back('n'); }
                else repl.push_back(c);
            }
            JParser p2;
            p2.in = repl;
            root = JValue();
            if (!p2.parse_document(root)) { d.err = EG_JSON; return d; }
        }
    }
    if (root.t != JValue::Object) { d.err = EG_EMPTY; return d; }  // :50
    StructuredData sd;
    std::optional<double> ts;
    std::optional<std::string> hostname, msg, full_msg;
    std::optional<uint8_t> severity;
    for (auto& kv : root.obj) {  // sorted-key order :51
        const std::string& key = kv.first;
        JValue& v = kv.second;
        if (key == "timestamp") {  // as_f64 :53
            if (v.t == JValue::I64) ts = (double)v.i;
            else if (v.t == JValue::U64) ts = (double)v.u;
            else if (v.t == JValue::F64) ts = v.f;
            else { d.err = EG_TS; return d; }
        } else if (key == "host") {
            if (v.t != JValue::String) { d.err = EG_HOST; return d; }
            hostname = v.s;
        } else if (key == "short_message") {
            if (v.t != JValue::String) { d.err = EG_SHORT; return d; }
            msg = v.s;
        } else if (key == "full_message") {
            if (v.t != JValue::String) { d.err = EG_FULL; return d; }
            full_msg = v.s;
        } else if (key == "version") {
            if (v.t != JValue::String) { d.err = EG_VERSION_T; return d; }
            if (v.s != "1.0" && v.s != "1.1") { d.err = EG_VERSION; return d; }
        } else if (key == "level") {  // as_u64 :83
            uint64_t sev;
            if (v.t == JValue::U64) sev = v.u;
            else if (v.t == JValue::I64 && v.i >= 0) sev = (uint64_t)v.i;
            else { d.err = EG_SEV; return d; }
            if (sev > 7) { d.err = EG_SEV_HIGH; return d; }
            severity = (uint8_t)sev;
        } else {
            SDValue sv;
            switch (v.t) {
                case JValue::String: sv.tag = SDTag::String; sv.s = v.s; break;
                case JValue::Bool: sv.tag = SDTag::Bool; sv.b = v.b; break;
                case JValue::F64: sv.tag = SDTag::F64; sv.f = v.f; break;
                case JValue::I64: sv.tag = SDTag::I64; sv.i = v.i; break;
                case JValue::U64: sv.tag = SDTag::U64; sv.u = v.u; break;
                case JValue::Null: sv.tag = SDTag::Null; break;
                default: d.err = EG_SD_TYPE; return d;  // :97
            }
            std::string name = (!key.empty() && key[0] == '_') ? key : "_" + key;
            sd.pairs.emplace_back(std::move(name), std::move(sv));
        }
    }
    if (!hostname) { d.err = EG_MISSING_HOST; return d; }  // :110 (ts default evaluated first, no error)
    if (ts) d.rec.ts = *ts;
    else d.ts_is_now = true;  // :109 PreciseTimestamp::now()
    d.rec.hostname = std::move(*hostname);
    d.rec.severity = severity;
    if (!sd.pairs.empty()) {
        std::vector<StructuredData> v;
        v.push_back(std::move(sd));
        d.rec.sd = std::move(v);
    }
    d.rec.msg = std::move(msg);
    d.rec.full_msg = std::move(full_msg);
    return d;
}

// ---------------------------------------------------------------------------
// Canonical dump + Rust Debug/Display renderings
// ---------------------------------------------------------------------------

static void put_s(std::string& o, std::string_view s) {
    char b[24];
    int n = snprintf(b, sizeof b, "%zu:", s.size());
    o.append(b, (size_t)n);
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
    int n = snprintf(b, sizeof b, "%016" PRIx64, bits);
    o.append(b, (size_t)n);
}

void dump(const Decoded& d, std::string& o) {
    char b[48];
    if (d.err) {
        o.append("E:");
        o.append(d.err);
    } else {
        const Record& r = d.rec;
        o.append("R:ts=");
        if (d.ts_is_now) o.append("now");
        else put_hex(o, r.ts);
        o.append(";fac=");
        if (r.facility) o.append(b, (size_t)snprintf(b, sizeof b, "%u", *r.facility)); else o.push_back('~');
        o.append(";sev=");
        if (r.severity) o.append(b, (size_t)snprintf(b, sizeof b, "%u", *r.severity)); else o.push_back('~');
        o.append(";host="); put_s(o, r.hostname);
        o.append(";app="); put_o(o, r.appname);
        o.append(";proc="); put_o(o, r.procid);
        o.append(";msgid="); put_o(o, r.msgid);
        o.append(";msg="); put_o(o, r.msg);
        o.append(";full="); put_o(o, r.full_msg);
        o.append(";sd=");
        if (!r.sd) o.push_back('~');
        else {
            o.append(b, (size_t)snprintf(b, sizeof b, "%zu", r.sd->size()));
            for (const auto& sd : *r.sd) {
                o.append("[id="); put_o(o, sd.sd_id);
                o.append(b, (size_t)snprintf(b, sizeof b, ";n=%zu", sd.pairs.size()));
                for (const auto& kv : sd.pairs) {
                    o.append(";k="); put_s(o, kv.first);
                    o.append(";v=");
                    const SDValue& v = kv.second;
                    switch (v.tag) {
                        case SDTag::String: o.push_back('s'); put_s(o, v.s); break;
                        case SDTag::Bool: o.append(v.b ? "b1" : "b0"); break;
                        case SDTag::F64: o.push_back('f'); put_hex(o, v.f); break;
                        case SDTag::I64: o.append(b, (size_t)snprintf(b, sizeof b, "i%" PRId64, v.i)); break;
                        case SDTag::U64: o.append(b, (size_t)snprintf(b, sizeof b, "u%" PRIu64, v.u)); break;
                        case SDTag::Null: o.push_back('n'); break;
                    }
                }
                o.push_back(']');
            }
        }
    }
    o.append(b, (size_t)snprintf(b, sizeof b, ";out=%zu", d.stdout_lines.size()));
    for (const auto& s : d.stdout_lines) { o.push_back(';'); put_s(o, s); }
}

// Rust float formatting (shortest round-trip digits; `{}`/`{:?}` differ only in
// always printing ".0" for Debug of integral values and in the exponent thresholds)
static std::string rust_f64(double f, bool debug) {
    if (std::isnan(f)) return "NaN";
    if (std::isinf(f)) return f < 0 ? "-inf" : "inf";
    char buf[64];
    double a = std::fabs(f);
    if (debug && a != 0.0 && (a >= 1e16 || a < 1e-4)) {
        auto r = std::to_chars(buf, buf + sizeof buf, f, std::chars_format::scientific);
        std::string s(buf, r.ptr);
        // to_chars gives d.ddde+XX ; Rust prints d.ddde16 / 1e-7
        size_t e = s.find('e');
        std::string mant = s.substr(0, e), ex = s.substr(e + 1);
        int ev = atoi(ex.c_str());
        return mant + "e" + std::to_string(ev);
    }
    auto r = std::to_chars(buf, buf + sizeof buf, f, std::chars_format::fixed);
    std::string s(buf, r.ptr);
    if (debug && s.find('.') == std::string::npos) s += ".0";
    return s;
}
static std::string rust_str_debug(std::string_view s) {
    std::string o = "\"";
    for (char c : s) {
        switch (c) {
            case '"': o += "\\\""; break;
            case '\\': o += "\\\\"; break;
            case '\n': o += "\\n"; break;
            case '\r': o += "\\r"; break;
            case '\t': o += "\\t"; break;
            default: o.push_back(c);
        }
    }
    o.push_back('"');
    return o;
}
static std::string opt_str_debug(const std::optional<std::string>& s) {
    return s ? "Some(" + rust_str_debug(*s) + ")" : "None";
}
static std::string opt_u8_debug(const std::optional<uint8_t>& v) {
    return v ? "Some(" + std::to_string((unsigned)*v) + ")" : "None";
}
static std::string sdvalue_debug(const SDValue& v) {
    switch (v.tag) {
        case SDTag::String: return "String(" + rust_str_debug(v.s) + ")";
        case SDTag::Bool: return std::string("Bool(") + (v.b ? "true" : "false") + ")";
        case SDTag::F64: return "F64(" + rust_f64(v.f, true) + ")";
        case SDTag::I64: return "I64(" + std::to_string(v.i) + ")";
        case SDTag::U64: return "U64(" + std::to_string(v.u) + ")";
        default: return "Null";
    }
}
// record.rs:42-68
std::string sd_display(const StructuredData& sd) {
    std::string o = "[";
    if (sd.sd_id) o += *sd.sd_id;
    for (const auto& kv : sd.pairs) {
        std::string_view name = kv.first;
        if (!name.empty() && name[0] == '_') name.remove_prefix(1);
        const SDValue& v = kv.second;
        o.push_back(' ');
        o.append(name);
        switch (v.tag) {
            case SDTag::String: o += "=\"" + v.s + "\""; break;
            case SDTag::Bool: o += std::string("=\"") + (v.b ? "true" : "false") + "\""; break;
            case SDTag::F64: o += "=\"" + rust_f64(v.f, false) + "\""; break;
            case SDTag::I64: o += "=\"" + std::to_string(v.i) + "\""; break;
            case SDTag::U64: o += "=\"" + std::to_string(v.u) + "\""; break;
            case SDTag::Null: break;
        }
    }
    o.push_back(']');
    return o;
}
std::string sd_debug(const StructuredData& sd) {
    std::string o = "StructuredData { sd_id: " + opt_str_debug(sd.sd_id) + ", pairs: [";
    bool first = true;
    for (const auto& kv : sd.pairs) {
        if (!first) o += ", ";
        first = false;
        o += "(" + rust_str_debug(kv.first) + ", " + sdvalue_debug(kv.second) + ")";
    }
    o += "] }";
    return o;
}
std::string record_debug(const Record& r) {
    std::string o = "Record { ts: " + rust_f64(r.ts, true) + ", hostname: " + rust_str_debug(r.hostname) +
                    ", facility: " + opt_u8_debug(r.facility) + ", severity: " + opt_u8_debug(r.severity) +
                    ", appname: " + opt_str_debug(r.appname) + ", procid: " + opt_str_debug(r.procid) +
                    ", msgid: " + opt_str_debug(r.msgid) + ", msg: " + opt_str_debug(r.msg) +
                    ", full_msg: " + opt_str_debug(r.full_msg) + ", sd: ";
    if (!r.sd) o += "None";
    else {
        o += "Some([";
        bool first = true;
        for (const auto& sd : *r.sd) {
            if (!first) o += ", ";
            first = false;
            o += sd_debug(sd);
        }
        o += "])";
    }
    o += " }";
    return o;
}

}  // namespace fgo
