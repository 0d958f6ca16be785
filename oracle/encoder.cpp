// oracle/encoder.cpp — TEST INFRASTRUCTURE, NOT PRODUCT CODE (see oracle.hpp).
//
// CPU restatement of the reference's GELF encoder, the stage that follows Decoder::decode in every splitter
// (splitter/line_splitter.rs:50-52):
//     GelfEncoder::encode      flowgger src/flowgger/encoder/gelf_encoder.rs:59-115
//     GelfEncoder::new         gelf_encoder.rs:29-48 (output.gelf_extra)
// The JSON text comes from un-vendored crates pinned in Cargo.toml: serde_json "~0.8" (`to_vec` over
// Value::Object(BTreeMap<String, Value>): keys in byte order, last insert wins, compact separators) and its float
// writer dtoa 0.2 (Grisu2 + prettify).  Both are restated here from their published algorithms:
//   * strings: serde_json 0.8 ser.rs `escape_bytes` escapes exactly `"` `\\` \b \f \n \r \t; every other byte —
//     including the remaining control bytes — is copied through  (PARITY UNPINNED: the reference's tests only show
//     `\n`; generators never emit other control bytes);
//   * U64/I64: decimal; Bool / Null: literals; F64: NaN and infinities -> `null`, else dtoa (PARITY UNPINNED beyond
//     the two values of gelf_encoder.rs:125,215).
// Pinned against the reference's own encoder tests (gelf_encoder.rs:125,152,175,215) in tests/test_oracle_golden.py.
#include <cinttypes>
#include <cmath>
#include <vector>
#include <cstdio>
#include <cstring>
#include <map>

#include "oracle.hpp"

namespace fgo {

namespace {

// ---- dtoa 0.2 (port of RapidJSON dtoa.h): Grisu2 ---------------------------------------------------------------
struct DiyFp {
    uint64_t f;
    int e;
};
DiyFp mul(DiyFp a, DiyFp b) {
    const unsigned __int128 p = (unsigned __int128)a.f * b.f;
    uint64_t h = (uint64_t)(p >> 64);
    const uint64_t l = (uint64_t)p;
    if (l & (1ull << 63)) ++h;  // mult_round
    return {h, a.e + b.e + 64};
}
// 10^k for k = -348 + 8 i as a 64-bit significand (rounded to nearest) and binary exponent, computed exactly here with
// 128-bit + big-number arithmetic instead of being copied from a table
struct Big {  // little-endian base 2^32 magnitude
    std::vector<uint32_t> d;
    void mul_small(uint32_t m) {
        uint64_t c = 0;
        for (auto& x : d) { c += (uint64_t)x * m; x = (uint32_t)c; c >>= 32; }
        if (c) d.push_back((uint32_t)c);
    }
    int bits() const {
        if (d.empty()) return 0;
        return (int)(d.size() - 1) * 32 + (32 - __builtin_clz(d.back()));
    }
    bool bit(int i) const { return i >= 0 && (size_t)(i / 32) < d.size() && ((d[(size_t)(i / 32)] >> (i % 32)) & 1u); }
    uint64_t top64(int from) const {  // bits [from-63, from]
        uint64_t v = 0;
        for (int i = 0; i < 64; ++i) v = (v << 1) | (bit(from - i) ? 1u : 0u);
        return v;
    }
    bool any_below(int i) const {
        for (int k = 0; k < i; ++k)
            if (bit(k)) return true;
        return false;
    }
};
DiyFp cached_power(int k10) {
    if (k10 >= 0) {
        Big b;
        b.d = {1};
        for (int i = 0; i < k10; ++i) b.mul_small(10);
        const int nb = b.bits();
        uint64_t f = b.top64(nb - 1);
        int e = nb - 64;
        if (b.bit(nb - 65)) {  // round to nearest (half up)
            if (++f == 0) { f = 1ull << 63; ++e; }
        }
        return {f, e};
    }
    // 10^-n = 2^s / 10^n: long division of 2^s by 10^n with s large enough for 64 quotient bits + a rounding bit
    const int n = -k10;
    Big den;
    den.d = {1};
    for (int i = 0; i < n; ++i) den.mul_small(10);
    const int s = den.bits() + 66;
    // quotient q = floor(2^s / den) has 66 or 67 bits: schoolbook bit-by-bit division on a remainder Big
    Big rem;
    rem.d = {0};
    std::vector<int> qbits;
    auto shl1_add = [&](Big& r, int bit) {
        uint32_t c = (uint32_t)bit;
        for (auto& x : r.d) { const uint32_t nc = x >> 31; x = (x << 1) | c; c = nc; }
        if (c) r.d.push_back(c);
    };
    auto ge = [&](const Big& a, const Big& b2) {
        size_t na = a.d.size(), nb = b2.d.size();
        while (na > 0 && a.d[na - 1] == 0) --na;
        while (nb > 0 && b2.d[nb - 1] == 0) --nb;
        if (na != nb) return na > nb;
        for (size_t i = na; i-- > 0;)
            if (a.d[i] != b2.d[i]) return a.d[i] > b2.d[i];
        return true;
    };
    auto sub = [&](Big& a, const Big& b2) {
        int64_t c = 0;
        for (size_t i = 0; i < a.d.size(); ++i) {
            int64_t v = (int64_t)a.d[i] - (i < b2.d.size() ? (int64_t)b2.d[i] : 0) + c;
            c = v < 0 ? -1 : 0;
            a.d[i] = (uint32_t)(v & 0xFFFFFFFFll);
        }
    };
    for (int i = s; i >= 0; --i) {
        shl1_add(rem, i == s ? 1 : 0);
        if (ge(rem, den)) { sub(rem, den); qbits.push_back(1); }
        else qbits.push_back(0);
    }
    size_t first = 0;
    while (first < qbits.size() && !qbits[first]) ++first;
    uint64_t f = 0;
    for (size_t i = 0; i < 64; ++i) f = (f << 1) | (uint64_t)qbits[first + i];
    int e = (int)(qbits.size() - first) - 64 - s;  // value = q * 2^-s, q has (size-first) bits
    if (qbits[first + 64]) {
        if (++f == 0) { f = 1ull << 63; ++e; }
    }
    return {f, e};
}
const DiyFp* power_table() {
    static DiyFp t[87];
    static bool init = false;
    if (!init) {
        for (int i = 0; i < 87; ++i) t[i] = cached_power(-348 + 8 * i);
        init = true;
    }
    return t;
}

void grisu_round(char* buf, int len, uint64_t delta, uint64_t rest, uint64_t ten_kappa, uint64_t wp_w) {
    while (rest < wp_w && delta - rest >= ten_kappa && (rest + ten_kappa < wp_w || wp_w - rest > rest + ten_kappa - wp_w)) {
        buf[len - 1]--;
        rest += ten_kappa;
    }
}
int grisu2(double value, char* buf, int* K) {
    static const uint32_t kPow10[] = {1, 10, 100, 1000, 10000, 100000, 1000000, 10000000, 100000000, 1000000000};
    uint64_t bits;
    memcpy(&bits, &value, 8);
    const int be = (int)((bits >> 52) & 0x7FF);
    const uint64_t fr = bits & ((1ull << 52) - 1);
    DiyFp v = be ? DiyFp{fr + (1ull << 52), be - 0x433} : DiyFp{fr, 1 - 0x433};
    DiyFp pl{(v.f << 1) + 1, v.e - 1};
    while (!(pl.f & (1ull << 53))) { pl.f <<= 1; --pl.e; }
    pl.f <<= 10;
    pl.e -= 10;
    DiyFp mi = v.f == (1ull << 52) ? DiyFp{(v.f << 2) - 1, v.e - 2} : DiyFp{(v.f << 1) - 1, v.e - 1};
    mi.f <<= mi.e - pl.e;
    mi.e = pl.e;
    const double dk = (double)(-61 - pl.e) * 0.30102999566398114 + 347.0;
    int k = (int)dk;
    if (dk - k > 0.0) ++k;
    const int index = (k >> 3) + 1;
    *K = -(-348 + (index << 3));
    const DiyFp c = power_table()[index];
    DiyFp vn = v;
    while (!(vn.f & (1ull << 63))) { vn.f <<= 1; --vn.e; }
    const DiyFp W = mul(vn, c);
    DiyFp Wp = mul(pl, c), Wm = mul(mi, c);
    ++Wm.f;
    --Wp.f;
    uint64_t delta = Wp.f - Wm.f;
    const DiyFp one{1ull << -Wp.e, Wp.e};
    const uint64_t wp_w = Wp.f - W.f;
    uint32_t p1 = (uint32_t)(Wp.f >> -one.e);
    uint64_t p2 = Wp.f & (one.f - 1);
    int kappa = 1;
    while (kappa < 10 && p1 >= kPow10[kappa]) ++kappa;
    int len = 0;
    while (kappa > 0) {
        const uint32_t d = p1 / kPow10[kappa - 1];
        p1 %= kPow10[kappa - 1];
        if (d || len) buf[len++] = (char)('0' + d);
        --kappa;
        const uint64_t tmp = ((uint64_t)p1 << -one.e) + p2;
        if (tmp <= delta) {
            *K += kappa;
            grisu_round(buf, len, delta, tmp, (uint64_t)kPow10[kappa] << -one.e, wp_w);
            return len;
        }
    }
    for (;;) {
        p2 *= 10;
        delta *= 10;
        const char d = (char)(p2 >> -one.e);
        if (d || len) buf[len++] = (char)('0' + d);
        p2 &= one.f - 1;
        --kappa;
        if (p2 < delta) {
            *K += kappa;
            const int idx = -kappa;
            grisu_round(buf, len, delta, p2, one.f, wp_w * (idx < 9 ? kPow10[idx] : 0));
            return len;
        }
    }
}
void write_f64(double value, std::string& o) {
    if (value != value || value == 1.0 / 0.0 || value == -1.0 / 0.0) {  // serde_json 0.8: non-finite -> null
        o += "null";
        return;
    }
    if (value == 0.0) {
        o += std::signbit(value) ? "-0.0" : "0.0";
        return;
    }
    if (value < 0.0) { o.push_back('-'); value = -value; }
    char dig[32];
    int k;
    const int length = grisu2(value, dig, &k);
    const int kk = length + k;
    std::string d(dig, (size_t)length);
    if (0 <= k && kk <= 21) o += d + std::string((size_t)(kk - length), '0') + ".0";
    else if (0 < kk && kk <= 21) o += d.substr(0, (size_t)kk) + "." + d.substr((size_t)kk);
    else if (-6 < kk && kk <= 0) o += "0." + std::string((size_t)(-kk), '0') + d;
    else {
        o += d.substr(0, 1);
        if (length > 1) o += "." + d.substr(1);
        o += "e" + std::to_string(kk - 1);
    }
}

// serde_json 0.8 ser.rs escape_bytes
void write_str(std::string_view s, std::string& o) {
    o.push_back('"');
    for (const char c : s) {
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

struct JVal {
    int kind = 0;  // 0 string 1 bool 2 f64 3 i64 4 u64 5 null
    std::string s;
    bool b = false;
    double f = 0;
    int64_t i = 0;
    uint64_t u = 0;
};
JVal jstr(std::string v) {
    JVal j;
    j.kind = 0;
    j.s = std::move(v);
    return j;
}

}  // namespace

std::string format_f64_json(double v) {
    std::string o;
    write_f64(v, o);
    return o;
}

// gelf_encoder.rs:59-115
std::string gelf_encode(const Record& record, const std::vector<std::pair<std::string, std::string>>& extra) {
    std::map<std::string, JVal> map;  // BTreeMap<String, Value>: byte order, insert replaces
    map["version"] = jstr("1.1");
    map["host"] = jstr(record.hostname.empty() ? "unknown" : record.hostname);
    map["short_message"] = jstr(record.msg ? *record.msg : "-");
    {
        JVal t;
        t.kind = 2;
        t.f = record.ts;
        map["timestamp"] = t;
    }
    if (record.severity) {
        JVal l;
        l.kind = 4;
        l.u = *record.severity;
        map["level"] = l;
    }
    if (record.full_msg) map["full_message"] = jstr(*record.full_msg);
    if (record.appname) map["application_name"] = jstr(*record.appname);
    if (record.procid) map["process_id"] = jstr(*record.procid);
    if (record.sd) {
        for (const auto& sd : *record.sd) {
            if (sd.sd_id) map["sd_id"] = jstr(*sd.sd_id);
            for (const auto& kv : sd.pairs) {
                JVal v;
                v.kind = (int)kv.second.tag;
                v.s = kv.second.s;
                v.b = kv.second.b;
                v.f = kv.second.f;
                v.i = kv.second.i;
                v.u = kv.second.u;
                map[kv.first] = v;
            }
        }
    }
    for (const auto& kv : extra) map[kv.first] = jstr(kv.second);
    std::string o = "{";
    bool first = true;
    char nb[32];
    for (const auto& kv : map) {
        if (!first) o.push_back(',');
        first = false;
        write_str(kv.first, o);
        o.push_back(':');
        const JVal& v = kv.second;
        switch (v.kind) {
            case 0: write_str(v.s, o); break;
            case 1: o += v.b ? "true" : "false"; break;
            case 2: write_f64(v.f, o); break;
            case 3: o.append(nb, (size_t)snprintf(nb, sizeof nb, "%" PRId64, v.i)); break;
            case 4: o.append(nb, (size_t)snprintf(nb, sizeof nb, "%" PRIu64, v.u)); break;
            default: o += "null";
        }
    }
    o.push_back('}');
    return o;
}

}  // namespace fgo
