// oracle/rfc3164.cpp — TEST INFRASTRUCTURE, NOT PRODUCT CODE (see oracle.hpp).
//
// CPU restatement of RFC3164Decoder::decode (flowgger src/flowgger/decoder/rfc3164_decoder.rs:31-213), written
// the way the reference is: owned token vectors, the "standard" form first, the "custom" form second.
//
// Un-vendored crates on this path, restated from their published behaviour:
//   time 0.3      format description "[year] [month repr:short] [day padding:none] [hour]:[minute]:[second]"
//                 (rfc3164_decoder.rs:187-190): optional sign + exactly 4 digits, a case-sensitive English month
//                 abbreviation, 1-2 digits (non-zero), three 2-digit fields; Date::from_calendar_date /
//                 Time::from_hms range checks; trailing input is an error.
//   time-tz 0.3   timezones::get_by_name (:196) = exact IANA name lookup; assume_timezone (:202) = the offset in force
//                 at that LOCAL time.  The zone table is handed in by the caller (tzread.py reads the system TZif files);
//                 a local time that exists twice takes the earlier offset, one that does not exist the offset before the
//                 jump — PARITY UNPINNED: no reference test covers either, time-tz's source is not available here.
// Pinned against the reference's own eleven tests (rfc3164_decoder.rs:218-425) in tests/test_oracle_golden.py.
#include <cstring>

#include "oracle.hpp"

namespace fgo {

static const char* const E3_PRI_MALFORMED = "Malformed RFC3164 event: Invalid priority";                         // :131
static const char* const E3_PRI_INVALID = "Invalid priority";                                                    // :137
static const char* const E3_STD = "Malformed RFC3164 standard event: Invalid timestamp or hostname";             // :85 (never final)
static const char* const E3_CUSTOM = "Malformed RFC3164 event: Invalid timestamp or hostname";                   // :120
static const char* const E3_TIME_FORMAT = "Invalid time format";                                                 // :158
static const char* const E3_WITH_YEAR = "Unable to parse RFC3164 date with year";                                // :178
static const char* const E3_DATE = "Unable to parse the date in RFC3164 decoder";                                // :211
const char* const E3_PANIC = "(the reference panics here: index out of bounds, rfc3164_decoder.rs:64)";

// char::is_whitespace on one decoded scalar (Unicode White_Space)
static bool is_white_space(uint32_t c) {
    return (c >= 0x09 && c <= 0x0D) || c == 0x20 || c == 0x85 || c == 0xA0 || c == 0x1680 || (c >= 0x2000 && c <= 0x200A) ||
           c == 0x2028 || c == 0x2029 || c == 0x202F || c == 0x205F || c == 0x3000;
}
// next scalar of valid UTF-8 at s[i]; advances i
static uint32_t next_char(std::string_view s, size_t& i) {
    const unsigned char c0 = (unsigned char)s[i];
    if (c0 < 0x80) { i += 1; return c0; }
    if (c0 < 0xE0 && i + 1 < s.size()) { uint32_t c = ((c0 & 0x1Fu) << 6) | ((unsigned char)s[i + 1] & 0x3Fu); i += 2; return c; }
    if (c0 < 0xF0 && i + 2 < s.size()) {
        uint32_t c = ((c0 & 0x0Fu) << 12) | (((unsigned char)s[i + 1] & 0x3Fu) << 6) | ((unsigned char)s[i + 2] & 0x3Fu);
        i += 3;
        return c;
    }
    if (i + 3 < s.size()) {
        uint32_t c = ((c0 & 0x07u) << 18) | (((unsigned char)s[i + 1] & 0x3Fu) << 12) | (((unsigned char)s[i + 2] & 0x3Fu) << 6) |
                     ((unsigned char)s[i + 3] & 0x3Fu);
        i += 4;
        return c;
    }
    i = s.size();
    return 0xFFFD;
}
// str::split_whitespace
static std::vector<std::string_view> split_whitespace(std::string_view s) {
    std::vector<std::string_view> v;
    size_t i = 0, start = 0;
    bool in = false;
    while (i < s.size()) {
        const size_t at = i;
        const uint32_t c = next_char(s, i);
        if (is_white_space(c)) {
            if (in) v.push_back(s.substr(start, at - start));
            in = false;
        } else if (!in) {
            in = true;
            start = at;
        }
    }
    if (in) v.push_back(s.substr(start));
    return v;
}
// str::split(": ")
static std::vector<std::string_view> split_str(std::string_view s, std::string_view sep) {
    std::vector<std::string_view> v;
    size_t a = 0;
    for (;;) {
        const size_t k = s.find(sep, a);
        if (k == std::string_view::npos) { v.push_back(s.substr(a)); return v; }
        v.push_back(s.substr(a, k - a));
        a = k + sep.size();
    }
}
static std::string join(const std::vector<std::string_view>& v, size_t from, size_t to, const char* sep) {
    std::string o;
    for (size_t k = from; k < to; ++k) {
        if (k > from) o += sep;
        o.append(v[k]);
    }
    return o;
}

static bool leap(int64_t y) { return (y % 4 == 0 && y % 100 != 0) || y % 400 == 0; }
static int month_days(int64_t y, int m) {
    static const int d[12] = {31, 28, 31, 30, 31, 30, 31, 31, 30, 31, 30, 31};
    return m == 2 && leap(y) ? 29 : d[m - 1];
}
static int64_t civil_days(int64_t y, int m, int d) {  // days since 1970-01-01, proleptic Gregorian
    y -= m <= 2;
    const int64_t era = (y >= 0 ? y : y - 399) / 400, yoe = y - era * 400;
    const int64_t doy = (153 * (m + (m > 2 ? -3 : 9)) + 2) / 5 + d - 1;
    return era * 146097 + yoe * 365 + yoe / 4 - yoe / 100 + doy - 719468;
}

// PrimitiveDateTime::parse(ts_str, "[year] [month repr:short] [day padding:none] [hour]:[minute]:[second]") -> seconds
// since the epoch of that civil time read as UTC
static bool parse_primitive(const std::string& s, int64_t& local) {
    static const char* MON[12] = {"Jan", "Feb", "Mar", "Apr", "May", "Jun", "Jul", "Aug", "Sep", "Oct", "Nov", "Dec"};
    size_t i = 0;
    auto digits = [&](int n, int64_t& out) {
        if (i + (size_t)n > s.size()) return false;
        int64_t v = 0;
        for (int k = 0; k < n; ++k) {
            const unsigned d = (unsigned char)s[i + (size_t)k] - '0';
            if (d > 9) return false;
            v = v * 10 + d;
        }
        i += (size_t)n;
        out = v;
        return true;
    };
    auto lit = [&](char c) {
        if (i < s.size() && s[i] == c) { ++i; return true; }
        return false;
    };
    bool neg = false;
    if (i < s.size() && (s[i] == '+' || s[i] == '-')) { neg = s[i] == '-'; ++i; }  // [year] sign:automatic
    int64_t year, day, hh, mm, ss;
    if (!digits(4, year)) return false;  // padding:zero, exactly four digits (large-dates is off)
    if (neg) year = -year;
    if (!lit(' ')) return false;
    int month = 0;
    for (int m = 0; m < 12; ++m)
        if (s.compare(i, 3, MON[m]) == 0) { month = m + 1; break; }
    if (!month) return false;
    i += 3;
    if (!lit(' ')) return false;
    if (i >= s.size() || s[i] < '0' || s[i] > '9') return false;  // [day padding:none]: 1..2 digits, greedy, NonZeroU8
    day = s[i++] - '0';
    if (i < s.size() && s[i] >= '0' && s[i] <= '9') day = day * 10 + (s[i++] - '0');
    if (day == 0) return false;
    if (!lit(' ') || !digits(2, hh) || !lit(':') || !digits(2, mm) || !lit(':') || !digits(2, ss)) return false;
    if (i != s.size()) return false;  // UnexpectedTrailingCharacters
    if (day > month_days(year, month)) return false;  // Date::from_calendar_date
    if (hh > 23 || mm > 59 || ss > 59) return false;  // Time::from_hms
    local = civil_days(year, month, (int)day) * 86400 + hh * 3600 + mm * 60 + ss;
    return true;
}

// utils/mod.rs:24-35: unix_timestamp_nanos() as f64 / 1e9
static double ts_of(int64_t unix_seconds) {
    const __int128 nanos = (__int128)unix_seconds * 1000000000;
    return (double)nanos / 1e9;
}

// the offset in force at LOCAL second `local` (see the header for the two corner rules)
static int32_t offset_at_local(const TzZone& z, int64_t local) {
    const size_t n = z.trans.size();  // span k: offs[k], UTC range [trans[k-1], trans[k])
    for (size_t k = 0; k <= n; ++k) {
        const bool after_start = k == 0 || local >= z.trans[k - 1] + z.offs[k];
        const bool before_end = k == n || local < z.trans[k] + z.offs[k];
        if (after_start && before_end) return z.offs[k];  // the earliest span that contains it
    }
    for (size_t k = 0; k < n; ++k)  // in no span: skipped by the jump at trans[k]
        if (local >= z.trans[k] + z.offs[k] && local < z.trans[k] + z.offs[k + 1]) return z.offs[k];
    return z.offs[n];
}

struct DateOut {
    double ts = 0.0;
    size_t idx = 0;  // tokens consumed
};

// parse_date (:163-213)
static const char* parse_date(const Rfc3164Config& cfg, const std::vector<std::string_view>& tok, bool has_year, DateOut& out) {
    std::string ts_str;
    size_t idx;
    if (has_year) {
        idx = 4;
        if (tok.size() < idx) return E3_WITH_YEAR;
        ts_str = join(tok, 0, idx, " ");
    } else {
        idx = 3;
        if (tok.size() < idx) return "Unable to parse RFC3164 date without year";  // :181 (unreachable: parse_date_token checks)
        ts_str = std::to_string(cfg.year) + " " + join(tok, 0, idx, " ");
    }
    int64_t local;
    if (!parse_primitive(ts_str, local)) return E3_DATE;
    const TzZone* tz = nullptr;
    if (tok.size() > idx) {
        auto it = cfg.zones.find(std::string(tok[idx]));
        if (it != cfg.zones.end()) tz = &it->second;
    }
    if (tz) {
        out.ts = ts_of(local - offset_at_local(*tz, local));
        idx += 1;
    } else {
        out.ts = ts_of(local);
    }
    out.idx = idx;
    return nullptr;
}
// parse_date_token (:155-161)
static const char* parse_date_token(const Rfc3164Config& cfg, const std::vector<std::string_view>& tok, DateOut& out) {
    if (tok.size() < 3) return E3_TIME_FORMAT;
    if (parse_date(cfg, tok, false, out) == nullptr) return nullptr;
    return parse_date(cfg, tok, true, out);
}

Decoded rfc3164_decode(const Rfc3164Config& cfg, std::string_view line) {
    Decoded d;
    // parse_strip_pri (:126-153)
    std::string_view msg = line;
    std::optional<uint8_t> facility, severity;
    if (!line.empty() && line[0] == '<') {
        const size_t gt = line.find('>');
        if (gt == std::string_view::npos) { d.err = E3_PRI_MALFORMED; return d; }
        std::string_view pri = line.substr(0, gt + 1);
        while (!pri.empty() && pri.front() == '<') pri.remove_prefix(1);
        while (!pri.empty() && pri.back() == '>') pri.remove_suffix(1);
        uint8_t npri;
        if (!rust_parse_u8(pri, npri)) { d.err = E3_PRI_INVALID; return d; }
        facility = (uint8_t)(npri >> 3);
        severity = (uint8_t)(npri & 7);
        msg = line.substr(gt + 1);
    }
    auto fill = [&](double ts, std::string_view host, std::string message) {
        d.rec.ts = ts;
        d.rec.hostname = std::string(host);
        d.rec.facility = facility;
        d.rec.severity = severity;
        d.rec.msg = std::move(message);
        d.rec.full_msg = std::string(rust_trim_end(line));
    };
    // decode_rfc_standard (:55-87)
    {
        const std::vector<std::string_view> tok = split_whitespace(msg);
        if (tok.size() > 3) {
            DateOut o;
            if (parse_date_token(cfg, tok, o) == nullptr) {
                if (o.idx >= tok.size()) { d.err = E3_PANIC; return d; }  // `_log_tokens[0]` on an empty Vec (:64)
                fill(o.ts, tok[o.idx], join(tok, o.idx + 1, tok.size(), " "));
                return d;
            }
        }
        (void)E3_STD;
    }
    // decode_rfc_custom (:89-123)
    const std::vector<std::string_view> tok = split_str(msg, ": ");
    if (tok.size() <= 2) { d.err = E3_CUSTOM; return d; }
    DateOut o;
    if (const char* e = parse_date_token(cfg, split_whitespace(tok[1]), o)) { d.err = e; return d; }
    fill(o.ts, tok[0], join(tok, 2, tok.size(), ": "));
    return d;
}

}  // namespace fgo
