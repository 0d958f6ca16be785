// fg_ltsv.cuh — one LTSV line -> Record fields, on device.
//
// H100-native replacement for LTSVDecoder::decode
// (flowgger src/flowgger/decoder/ltsv_decoder.rs:87-221) and its helpers
// rfc3339_to_unix :224-229, english_time_to_unix[_with_subsecond] :231-254,
// unix_strtime_to_unix :256-261, parse_ts :263-267.  Schema / suffix configuration
// (LTSVDecoder::new :24-83) arrives as flat device arrays (LtsvDeviceConfig).
//
// Lock-step discipline as in fg_rfc5424.cuh: one outer iteration = one tab-separated part per
// lane; the byte scans inside are warp-uniform `lim`-bounded loops.
#pragma once
#include "fg_common.cuh"
#include "fg_float.cuh"
#include "fg_kernels.cuh"
#include "fg_rfc5424.cuh"
#include "fg_status.h"

namespace fg {

// "[day padding:none]/[month repr:short]/[year]:[hour]:[minute]:[second](.[subsecond]) [offset_hour sign:mandatory][offset_minute]"
// (ltsv_decoder.rs:239-247), `time` 0.3 format-description semantics.
static __device__ __noinline__ bool parse_english_time(bytes_t p, int a, int b, bool with_subsecond, double& ts) {
    int i = a;
    DateTime t;
    t.nanos = 0;
    if (i >= b || !is_digit(p[i])) return false;
    t.day = (int)(p[i++] - '0');
    if (i < b && is_digit(p[i])) t.day = t.day * 10 + (int)(p[i++] - '0');
    if (t.day == 0) return false;  // NonZeroU8
    if (i >= b || p[i] != '/') return false;
    ++i;
    if (i + 3 > b) return false;
    {
        const uint32_t m3 = ((uint32_t)p[i] << 16) | ((uint32_t)p[i + 1] << 8) | (uint32_t)p[i + 2];
        int m = 0;
        switch (m3) {  // case-sensitive short month names
            case 0x4A616E: m = 1; break;   // Jan
            case 0x466562: m = 2; break;   // Feb
            case 0x4D6172: m = 3; break;   // Mar
            case 0x417072: m = 4; break;   // Apr
            case 0x4D6179: m = 5; break;   // May
            case 0x4A756E: m = 6; break;   // Jun
            case 0x4A756C: m = 7; break;   // Jul
            case 0x417567: m = 8; break;   // Aug
            case 0x536570: m = 9; break;   // Sep
            case 0x4F6374: m = 10; break;  // Oct
            case 0x4E6F76: m = 11; break;  // Nov
            case 0x446563: m = 12; break;  // Dec
            default: return false;
        }
        t.month = m;
        i += 3;
    }
    if (i >= b || p[i] != '/') return false;
    ++i;
    bool yneg = false;
    if (i < b && (p[i] == '+' || p[i] == '-')) { yneg = p[i] == '-'; ++i; }
    if (!four_digits(p, i, b, t.year)) return false;
    if (yneg) t.year = -t.year;
    if (i >= b || p[i] != ':') return false;
    ++i;
    if (!two_digits(p, i, b, t.hour)) return false;
    if (i >= b || p[i] != ':') return false;
    ++i;
    if (!two_digits(p, i, b, t.minute)) return false;
    if (i >= b || p[i] != ':') return false;
    ++i;
    if (!two_digits(p, i, b, t.second)) return false;
    if (with_subsecond) {
        if (i >= b || p[i] != '.') return false;
        ++i;
        if (!subsecond(p, i, b, t.nanos)) return false;
    }
    if (i >= b || p[i] != ' ') return false;
    ++i;
    if (i >= b || (p[i] != '+' && p[i] != '-')) return false;  // sign:mandatory
    const bool oneg = p[i] == '-';
    ++i;
    int oh, om;
    if (!two_digits(p, i, b, oh) || !two_digits(p, i, b, om)) return false;
    if (oh > 25 || om > 59) return false;
    t.offset_seconds = (oh * 3600 + om * 60) * (oneg ? -1 : 1);
    if (i != b) return false;
    return finish_datetime(t, false, ts);  // second == 60 is out of range for custom formats
}

// parse_ts :263-267: f64::from_str, then RFC3339, then the two English forms
static __device__ __noinline__ bool ltsv_parse_ts(bytes_t p, int a, int b, double& ts) {
    if (parse_f64_rust(p, a, b, ts)) return true;
    if (parse_rfc3339(p, a, b, ts)) return true;
    if (parse_english_time(p, a, b, false, ts)) return true;
    return parse_english_time(p, a, b, true, ts);
}

FG_DEV bool key_is(bytes_t p, int a, int n, const char* lit, int litn) {
    if (n != litn) return false;
    for (int k = 0; k < litn; ++k)
        if (p[a + k] != (uint8_t)lit[k]) return false;
    return true;
}

// schema.get(name) :129 — linear scan of the (small) configured key set; returns the fg_ltsv_type or 0 (string)
static __device__ __noinline__ int ltsv_schema_type(bytes_t p, int a, int n, const LtsvDeviceConfig& cfg) {
    for (int k = 0; k < cfg.n_schema; ++k) {
        const int o = cfg.name_off[k], l = cfg.name_off[k + 1] - o;
        if (l != n) continue;
        bool eq = true;
        for (int j = 0; j < n && eq; ++j) eq = cfg.names[o + j] == p[a + j];
        if (eq) return cfg.types[k];
    }
    return 0;
}
// !name.ends_with(suffix) :131 etc.
static __device__ __noinline__ bool ltsv_needs_suffix(bytes_t p, int a, int n, int type, const LtsvDeviceConfig& cfg) {
    if (!((cfg.suffix_present >> type) & 1u)) return false;
    const int o = cfg.suffix_off[type], l = cfg.suffix_off[type + 1] - o;
    if (l > n) return true;
    for (int j = 0; j < l; ++j)
        if (cfg.suffix[o + j] != p[a + n - l + j]) return true;
    return false;
}


// typed value of a schema key (:138-195): returns FG_ST_OK and the 8 value bytes, or the reference's type error
static __device__ __noinline__ uint32_t ltsv_parse_typed(bytes_t p, int va, int vb, int type, unsigned long long& val) {
    if (type == 1) {  // bool::from_str: exactly "true" / "false"
        if (key_is(p, va, vb - va, "true", 4)) { val = 1; return FG_ST_OK; }
        if (key_is(p, va, vb - va, "false", 5)) { val = 0; return FG_ST_OK; }
        return FG_EL_BOOL;
    }
    if (type == 2) {
        double f;
        if (!parse_f64_rust(p, va, vb, f)) return FG_EL_F64;
        val = (unsigned long long)__double_as_longlong(f);
        return FG_ST_OK;
    }
    if (type == 3) {
        int64_t v;
        if (!parse_i64(p, va, vb, v)) return FG_EL_I64;
        val = (unsigned long long)v;
        return FG_ST_OK;
    }
    uint64_t v;
    if (!parse_u64(p, va, vb, v)) return FG_EL_U64;
    val = v;
    return FG_ST_OK;
}

// All 32 lanes of a warp must call this (idle lanes with len = 0, active_line = false).
FG_DEV void ltsv_parse_line(bytes_t p, int len, int line_off, uint32_t sbase, bool active_line,
                            const LtsvDeviceConfig& cfg, LineResult& r, const EntrySink& sink) {
    r.ts = 0.0;
    r.facility = 0xFFu;
    r.severity = 0xFFu;
    r.flags = 0;
    r.host_o = r.app_o = r.proc_o = r.mid_o = r.msg_o = r.full_o = -1;
    r.host_l = r.app_l = r.proc_l = r.mid_l = r.msg_l = r.full_l = 0;
    r.n_entries = 0;
    uint32_t status = FG_ST_OK, n = 0, flags = 0;
    bool have_ts = false;
    int err_pos = 0;
    int part = 0;  // start of the current part
    bool active = active_line;
    const uint32_t b0 = (uint32_t)(size_t)p & 15u;
    const uint4* qp = (const uint4*)(p - b0);
    // The `time` value is parsed AFTER the part loop, in lock step for the whole warp (its position among the 20
    // fields differs per line, so parsing it inline would run one lane at a time).  Evaluation order is preserved:
    // a second `time`, or any error found later in the line, first settles the pending one.
    int ts_a = -1, ts_b = -1, ts_part = 0;
    bool err_set = false;
    uint32_t np = 0;  // parked typed values
    int t_va0 = 0, t_va1 = 0, t_va2 = 0, t_va3 = 0, t_pt0 = 0, t_pt1 = 0, t_pt2 = 0, t_pt3 = 0;
    uint32_t t_pk0 = 0, t_pk1 = 0, t_pk2 = 0, t_pk3 = 0;
    while (__any_sync(kFullMask, active)) {  // line.split('\t') :94
        // scan the part 16 bytes per step: first ':' (splitn(2, ':') :95), then the terminating TAB
        int i = part;
        {
            const int lim = active ? len : i;
            for (;;) {
                bool more = false;
                if (i < lim) {
                    bool hit;
                    i = scan_block16<true>(qp, b0, i, 0x09090909u, 0x3A3A3A3Au, hit);
                    more = !hit;
                }
                if (!__any_sync(kFullMask, more)) break;
            }
            if (i > len) i = len;  // a hit past the end of the line belongs to the next one
        }
        const bool has_colon = active && i < len && p[i] == ':';
        const int colon = i;
        {
            const int lim = has_colon ? len : i;
            for (;;) {
                bool more = false;
                if (i < lim) {
                    bool hit;
                    i = scan_block16<false>(qp, b0, i, 0x09090909u, 0u, hit);
                    more = !hit;
                }
                if (!__any_sync(kFullMask, more)) break;
            }
            if (i > len) i = len;
        }
        const int part_end = i;
        if (active) {
            if (!has_colon) {
                flags |= 0x02u;  // FG_FLAG_MISSING_VALUE: println! at :99 is replayed by the host
            } else {
                const int ka = part, kn = colon - part, va = colon + 1, vb = part_end;
                // the four reserved keys differ in (length, first byte): one cheap test rejects ordinary keys
                const uint32_t k0 = kn > 0 ? p[ka] : 0u;
                const bool maybe = (kn == 4 && (k0 == 't' || k0 == 'h')) || (kn == 7 && k0 == 'm') || (kn == 5 && k0 == 'l');
                if (maybe && key_is(p, ka, kn, "time", 4)) {  // :104-111
                    if (ts_a >= 0) {  // an earlier `time` is still pending: it is evaluated first (a failure returns there)
                        if (ltsv_parse_ts(p, ts_a, ts_b, r.ts)) have_ts = true;
                        else { status = FG_EL_TS; err_pos = ts_part; err_set = true; }
                    }
                    if (status == FG_ST_OK) {
                        ts_a = va;
                        ts_b = vb;
                        ts_part = part;
                        if (ts_b - ts_a >= 2 && p[ts_a] == '[' && p[ts_b - 1] == ']') { ++ts_a; --ts_b; }
                    } else {
                        ts_a = -1;
                    }
                } else if (maybe && key_is(p, ka, kn, "host", 4)) {
                    r.host_o = va;
                    r.host_l = vb - va;
                } else if (maybe && key_is(p, ka, kn, "message", 7)) {
                    r.msg_o = va;
                    r.msg_l = vb - va;
                } else if (maybe && key_is(p, ka, kn, "level", 5)) {  // :114-121
                    uint32_t sev;
                    if (!parse_u8(p, va, vb, sev)) status = FG_EL_SEV;
                    else if (sev > 7u) status = FG_EL_SEV_HIGH;
                    else r.severity = sev;
                } else {  // :122-199
                    const int type = cfg.has_schema ? ltsv_schema_type(p, ka, kn, cfg) : 0;
                    unsigned long long val = (unsigned long long)(uint32_t)(line_off + va) | ((unsigned long long)(uint32_t)(vb - va) << 32);
                    uint32_t meta = (uint32_t)type;  // FG_TAG_* == fg_ltsv_type
                    if (type != 0 && ltsv_needs_suffix(p, ka, kn, type, cfg)) meta |= 0x20u;  // FG_EM_SUFFIX
                    const uint32_t e = sbase + n;
                    bool deferred = false;
                    if (type != 0) {
                        // typed values sit at different field positions in every line: parsing them here would run one lane at a
                        // time, so up to 4 per line are parked in registers and parsed in lock step after the part loop
                        if (np < 4u && (vb - va) < (1 << 20) && n < 256u) {
                            const uint32_t packed = (uint32_t)(vb - va) | ((uint32_t)type << 20) | (n << 24);
                            if (np == 0u) { t_va0 = va; t_pk0 = packed; t_pt0 = part; }
                            else if (np == 1u) { t_va1 = va; t_pk1 = packed; t_pt1 = part; }
                            else if (np == 2u) { t_va2 = va; t_pk2 = packed; t_pt2 = part; }
                            else { t_va3 = va; t_pk3 = packed; t_pt3 = part; }
                            ++np;
                            deferred = true;
                        } else {
                            status = ltsv_parse_typed(p, va, vb, type, val);
                        }
                    }
                    if (status == FG_ST_OK) {
                        sink.name[e] = make_int2(line_off + ka, kn);
                        if (!deferred) sink.val[e] = val;
                        sink.meta[e] = (uint8_t)meta;
                        ++n;
                    }
                }
            }
            if (status != FG_ST_OK) {
                if (!err_set) err_pos = part;  // the error belongs to the current part (unless an earlier `time` already failed)
                active = false;
            } else if (part_end >= len) {
                active = false;
            } else {
                part = part_end + 1;
            }
        }
    }
    // Deferred work, in lock step.  All of it is pure, so it is evaluated even when a later part already failed; the
    // reference returns at the FIRST failing part, i.e. the candidate error with the smallest part position wins.
    {
        const bool pend = active_line && ts_a >= 0 && (status == FG_ST_OK || ts_part < err_pos);
        if (__any_sync(kFullMask, pend)) {
            if (pend) {
                double t;
                if (ltsv_parse_ts(p, ts_a, ts_b, t)) { r.ts = t; have_ts = true; }
                else { status = FG_EL_TS; err_pos = ts_part; }
            }
        }
    }
#pragma unroll
    for (uint32_t sl = 0; sl < 4u; ++sl) {
        const int va = sl == 0u ? t_va0 : (sl == 1u ? t_va1 : (sl == 2u ? t_va2 : t_va3));
        const uint32_t pk = sl == 0u ? t_pk0 : (sl == 1u ? t_pk1 : (sl == 2u ? t_pk2 : t_pk3));
        const int pt = sl == 0u ? t_pt0 : (sl == 1u ? t_pt1 : (sl == 2u ? t_pt2 : t_pt3));
        const bool has = active_line && sl < np && (status == FG_ST_OK || pt < err_pos);
        if (__any_sync(kFullMask, has)) {
            if (has) {
                unsigned long long val = 0;
                const uint32_t st = ltsv_parse_typed(p, va, va + (int)(pk & 0xFFFFFu), (int)((pk >> 20) & 7u), val);
                if (st == FG_ST_OK) sink.val[sbase + (pk >> 24)] = val;
                else { status = st; err_pos = pt; }
            }
        }
    }
    if (active_line && status == FG_ST_OK) {
        if (!have_ts) { status = FG_EL_MISSING_TS; err_pos = len + 1; }             // :205
        else if (r.host_o < 0) { status = FG_EL_MISSING_HOST; err_pos = len + 1; }  // :206
    }
    if (status == FG_ST_OK) {
        r.full_o = 0;  // full_msg = the whole line, untrimmed :219
        r.full_l = len;
        r.n_entries = n;
    } else {
        r.full_o = err_pos;
    }
    r.flags = flags;
    r.status = status;
    __syncwarp();
}

}  // namespace fg
