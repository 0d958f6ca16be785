// emu_ltsv.cpp — CPU emulation of the LTSV device logic (TEST INFRASTRUCTURE, see cuda_shim.h).
//
// Compiles the product's device sources (fg_ltsvfast.cuh: stage-1 TAB bitmap, lt_part, lt_finish_line; fg_ltsv.cuh: the
// value parsers and the direct-path scanner) with g++ and replays what parse_ltsv_kernel does with them — CTA rounds over
// a staging tile, one slot per tab-separated part, the per-part and per-line phases, side-table placement — one thread at a time.
// The result has the layout of fg_batch_out (columnar rows + side table), so the CPU test-suite can push it through the
// product's materialiser and compare with the oracle without a GPU.
#define FG_HOST_EMU 1
#include <algorithm>
#include <cstdlib>
#include <cstring>
#include <string>
#include <vector>

#include "../../include/flowgger_cuda.h"
#include "../../flowgger_b200/csrc/fg_ltsvfast.cuh"

namespace {
constexpr int kLines = fg::kLtsvLinesPerCta;
constexpr int kSlots = fg::kLtsvStageSlots;

struct Tables {
    std::vector<double> ts;
    std::vector<uint32_t> meta;
    std::vector<fg_span> host, msg, full, sd, none;
    std::vector<fg_span> ename;
    std::vector<uint64_t> eval;
    std::vector<uint8_t> emeta;
    int rounds = 0, direct = 0;
};

void put_row(Tables& t, int i, int o0, const fg::LineResult& res, uint32_t begin, uint32_t n) {
    const bool ok = res.status == FG_ST_OK;
    t.ts[i] = res.ts;
    t.meta[i] = res.status | (res.facility << 8) | (res.severity << 16) | (res.flags << 24);
    t.host[i] = fg_span{res.host_o >= 0 ? o0 + res.host_o : -1, res.host_l};
    t.msg[i] = fg_span{res.msg_o >= 0 ? o0 + res.msg_o : -1, res.msg_l};
    t.full[i] = ok ? fg_span{res.full_o >= 0 ? o0 + res.full_o : -1, res.full_l} : fg_span{o0 + std::max(res.full_o, 0), 0};
    t.sd[i] = fg_span{(int32_t)begin, (int32_t)n};
}
}  // namespace

extern "C" {

// stage 1's TAB mask of a 16-byte granule | (the ':' mask of its first 8 bytes, lt_colon_flags8, << 16): exposed so tests
// can pin the SWAR identities per byte
uint32_t emu_ltsv_classify16(const uint8_t* p) {
    uint32_t w[4], t, c;
    memcpy(w, p, 16);
    t = fg::lt_tab16(w[0], w[1], w[2], w[3]);
    unsigned long long k8;
    memcpy(&k8, p, 8);
    const unsigned long long z = fg::lt_colon_flags8(k8);
    c = 0;
    for (int b = 0; b < 8; ++b)
        if ((z >> (8 * b + 7)) & 1ull) c |= 1u << b;
    if (z && !((c >> fg::lt_first_flag8(z)) & 1u)) c = 0xFFFFu;  // the first-flag index must name a flagged byte
    if (z && (c & ((1u << fg::lt_first_flag8(z)) - 1u))) c = 0xFFFFu;  // ... the lowest one
    return t | (c << 16);
}

// schema: n_schema names (NUL-terminated) + types; suffix[5] indexed by fg_ltsv_type (nullptr = none)
int emu_ltsv_decode(const uint8_t* bytes, const int32_t* offsets, int32_t n, int32_t tile_bytes, int32_t strip_eol,
                    const uint8_t* invalid, int32_t has_schema, int32_t n_schema, const char* const* names, const int32_t* types,
                    const char* const* suffix, fg_batch_out* out, int32_t* info /* [3]: rounds, direct-path lines, schema staged */) {
    Tables* T = new Tables();
    const size_t nn = (size_t)std::max(n, 1);
    T->ts.resize(nn); T->meta.resize(nn); T->host.resize(nn); T->msg.resize(nn); T->full.resize(nn); T->sd.resize(nn);
    T->none.assign(nn, fg_span{-1, 0});
    // LtsvDeviceConfig, as fg_create lays it out
    std::string name_blob, suffix_blob;
    std::vector<int32_t> name_off{0}, tys;
    for (int k = 0; k < n_schema; ++k) {
        name_blob += names[k];
        name_off.push_back((int32_t)name_blob.size());
        tys.push_back(types[k]);
    }
    fg::LtsvDeviceConfig cfg{};
    cfg.has_schema = (has_schema || n_schema > 0) ? 1 : 0;
    cfg.n_schema = n_schema;
    cfg.suffix_off[0] = 0;
    for (int t = 0; t < 5; ++t) {
        if (t > 0 && suffix && suffix[t]) {
            cfg.suffix_present |= 1u << t;
            suffix_blob += suffix[t];
        }
        cfg.suffix_off[t + 1] = (int32_t)suffix_blob.size();
    }
    cfg.names = (const uint8_t*)name_blob.data();
    cfg.name_off = name_off.data();
    cfg.types = tys.data();
    cfg.suffix = (const uint8_t*)suffix_blob.data();
    const bool typed = cfg.has_schema != 0;
    uint32_t first[8], len_mask;
    fg::lt_schema_filters(cfg.names, cfg.name_off, cfg.n_schema, len_mask, first);
    // parse_ltsv_kernel stages a schema of <= 64 keys, <= 1024 name bytes and <= 64 suffix bytes in shared memory with the
    // two filters; a larger one is read from global memory with the filters off
    const bool staged = cfg.n_schema <= 64 && name_blob.size() <= 1024 && suffix_blob.size() <= 64;
    const fg::LtsvSchemaView S = {cfg.names, cfg.name_off, cfg.types, cfg.n_schema, staged ? len_mask : 0xFFFFFFFFu,
                                  staged ? first : nullptr};

    const int64_t total_bytes = n > 0 ? offsets[n] : 0;
    std::vector<uint8_t> tile((size_t)tile_bytes + 64);
    const int bm_words = tile_bytes / 32 + 4;
    std::vector<uint32_t> bmT((size_t)bm_words + 4);
    std::vector<unsigned long long> stage((size_t)kSlots), stage_val((size_t)kSlots);
    // scratch table of the direct path
    std::vector<fg_span> tname;
    std::vector<uint64_t> tval;
    std::vector<uint8_t> tmeta;

    auto direct_line = [&](int i) {
        ++T->direct;
        const int d0 = offsets[i];
        int len = offsets[i + 1] - d0;
        bool bad = false;
        if (strip_eol && len > 0) {
            len = fg::strip_terminator(bytes + d0, 0, len, strip_eol);
            if (invalid && invalid[i]) { bad = true; len = 0; }
        }
        tname.assign((size_t)len / 2 + 2, fg_span{0, 0});
        tval.assign(tname.size(), 0);
        tmeta.assign(tname.size(), 0);
        fg::EntrySink tmp = {(int2*)tname.data(), (unsigned long long*)tval.data(), tmeta.data()};
        fg::LineResult res;
        fg::ltsv_parse_line(bytes + d0, len, d0, 0u, true, cfg, res, tmp);
        if (bad) { res.status = FG_ES_INVALID_UTF8; res.n_entries = 0; res.full_o = 0; }
        const uint32_t my_n = res.status == FG_ST_OK ? res.n_entries : 0u;
        const uint32_t begin = my_n ? (uint32_t)T->ename.size() : 0u;
        for (uint32_t k = 0; k < my_n; ++k) {
            T->ename.push_back(tname[k]);
            T->eval.push_back(tval[k]);
            T->emeta.push_back(tmeta[k]);
        }
        put_row(*T, i, d0, res, begin, my_n);
    };

    for (int first = 0; first < n; first += kLines) {
        const int last = std::min(n, first + kLines);
        int cur = first;
        bool direct_next = false;
        while (cur < last) {
            const int base = fg::span_base(offsets[cur]);
            int r = 0;
            if (!direct_next)
                while (cur + r < last && offsets[cur + r + 1] - base <= tile_bytes) ++r;
            if (r == 0) {
                direct_next = false;
                direct_line(cur);
                ++cur;
                continue;
            }
            ++T->rounds;
            const uint32_t nbytes = fg::span_copy_bytes(base, offsets[cur + r]);
            for (uint32_t k = 0; k < nbytes; ++k) tile[k] = (int64_t)base + k < total_bytes ? bytes[base + k] : 0;  // the bulk copy
            const int nword = (int)((nbytes + 31u) >> 5);
            for (int g = 0; g < nword; ++g)
                bmT[g] = (emu_ltsv_classify16(tile.data() + 32 * g) & 0xFFFFu) | (emu_ltsv_classify16(tile.data() + 32 * g + 16) << 16);
            // (3) slots: one per part
            std::vector<int> ls((size_t)r), le((size_t)r);
            std::vector<uint32_t> nb((size_t)r), slot0((size_t)r);
            std::vector<char> bad((size_t)r, 0);
            uint32_t run = 0;
            int r2 = 0;
            for (int tid = 0; tid < r; ++tid) {
                const int i = cur + tid;
                ls[tid] = offsets[i] - base;
                le[tid] = offsets[i + 1] - base;
                if (strip_eol && le[tid] > ls[tid]) {
                    le[tid] = fg::strip_terminator(tile.data(), ls[tid], le[tid], strip_eol);
                    if (invalid && invalid[i]) bad[tid] = 1;
                }
                nb[tid] = bad[tid] ? 0u : (uint32_t)fg::lt_count_tabs(bmT.data(), ls[tid], le[tid]) + 1u;
                slot0[tid] = run;
                run += nb[tid];
                if (run <= (uint32_t)kSlots && r2 == tid) r2 = tid + 1;
            }
            if (r2 == 0) {
                direct_next = true;
                continue;
            }
            r = r2;
            std::vector<uint16_t> tabs((size_t)kSlots + 1);
            for (int tid = 0; tid < r; ++tid)
                if (!bad[tid]) fg::lt_list_tabs(bmT.data(), ls[tid], le[tid], tabs.data() + slot0[tid]);
            for (int tid = 0; tid < r; ++tid) {
                const int i = cur + tid;
                fg::LineResult res;
                res.ts = 0.0; res.facility = 0xFFu; res.severity = 0xFFu; res.flags = 0; res.status = FG_ST_OK;
                res.host_o = res.app_o = res.proc_o = res.mid_o = res.msg_o = res.full_o = -1;
                res.host_l = res.app_l = res.proc_l = res.mid_l = res.msg_l = res.full_l = 0;
                res.n_entries = 0;
                if (bad[tid]) {
                    res.status = FG_ES_INVALID_UTF8;
                    res.full_o = 0;
                    put_row(*T, i, offsets[i], res, 0, 0);
                    continue;
                }
                // (4) parts, (5) typed values
                uint32_t host_s = 0, msg_s = 0, time_s = 0, level_s = 0, ntime = 0, nlevel = 0, flags = 0, err = 0xFFFFFFFFu;
                for (uint32_t k = 0; k < nb[tid]; ++k) {
                    const uint32_t sl = slot0[tid] + k;
                    const int start = k == 0 ? ls[tid] : (int)tabs[sl - 1] + 1, end = (int)tabs[sl];
                    const fg::LtPart pt = typed ? fg::lt_part<true>(tile.data(), start, end, cfg, S) : fg::lt_part<false>(tile.data(), start, end, cfg, S);
                    stage[sl] = pt.row;
                    if (pt.kind == fg::LP_NONE) flags |= 0x02u;
                    else if (pt.kind == fg::LP_HOST) host_s = sl + 1;
                    else if (pt.kind == fg::LP_MSG) msg_s = sl + 1;
                    else if (pt.kind == fg::LP_TIME) { time_s = sl + 1; ++ntime; }
                    else if (pt.kind == fg::LP_LEVEL) { level_s = sl + 1; ++nlevel; }
                    const int type = (int)((pt.row >> 56) & 0x07u);
                    if (typed && type != 0) {
                        const int va = start + pt.kn + 1;
                        unsigned long long val = 0;
                        const uint32_t st = fg::ltsv_parse_typed(tile.data(), va, end, type, val);
                        if (st == FG_ST_OK) stage_val[sl] = val;
                        else err = std::min(err, (k << 8) | st);
                    }
                }
                if (ntime > 1 || nlevel > 1) {  // a repeated `time` / `level`: the round-1 scanner
                    direct_line(i);
                    continue;
                }
                auto value_of = [&](uint32_t s1, int key_len, int& a, int& b, int& k) {
                    a = -1; b = 0; k = 0;
                    if (s1 == 0u) return;
                    const uint32_t sl = s1 - 1u;
                    k = (int)(sl - slot0[tid]);
                    const int start = k == 0 ? ls[tid] : (int)tabs[sl - 1] + 1;
                    a = start + key_len + 1;
                    b = (int)tabs[sl];
                };
                int t_a, t_b, t_k, l_a, l_b, l_k, h_a, h_b, h_k, m_a, m_b, m_k;
                value_of(time_s, 4, t_a, t_b, t_k);
                value_of(level_s, 5, l_a, l_b, l_k);
                value_of(host_s, 4, h_a, h_b, h_k);
                value_of(msg_s, 7, m_a, m_b, m_k);
                double tsv = 0.0;
                bool ts_ok = false;
                if (t_a >= 0) {
                    (void)fg::lt_time_class(tile.data(), t_a, t_b);  // a scheduling hint on the device: must not fault on any value
                    ts_ok = fg::lt_time_value(tile.data(), t_a, t_b, tsv);
                }
                const int bad_k = fg::lt_finish_line(tile.data(), t_a >= 0 ? t_k : -1, ts_ok, tsv, l_a, l_b, l_k, err, h_a >= 0, res);
                res.flags = flags;
                if (res.status == FG_ST_OK) {
                    if (h_a >= 0) { res.host_o = h_a - ls[tid]; res.host_l = h_b - h_a; }
                    if (m_a >= 0) { res.msg_o = m_a - ls[tid]; res.msg_l = m_b - m_a; }
                    res.full_o = 0;
                    res.full_l = le[tid] - ls[tid];
                } else {
                    res.full_o = bad_k >= 0 ? (bad_k == 0 ? ls[tid] : (int)tabs[slot0[tid] + (uint32_t)bad_k - 1u] + 1) - ls[tid] : (le[tid] - ls[tid]) + 1;
                    res.severity = 0xFFu;
                    res.ts = 0.0;
                }
                // (6) the rows of the line, in slot order
                uint32_t my_n = 0;
                const uint32_t begin = (uint32_t)T->ename.size();
                if (res.status == FG_ST_OK) {
                    for (uint32_t k = 0; k < nb[tid]; ++k) {
                        const unsigned long long e = stage[slot0[tid] + k];
                        if (e == 0ull) continue;
                        const int ka = base + (int)(e & 0xFFFFu), kn = (int)((e >> 16) & 0xFFFFu);
                        const uint32_t meta = (uint32_t)(e >> 56) & 0x7Fu;
                        unsigned long long v = (unsigned long long)(uint32_t)(ka + kn + 1) | (((e >> 32) & 0xFFFFFFull) << 32);
                        if (typed && (meta & 0x07u) != 0u) v = stage_val[slot0[tid] + k];
                        T->ename.push_back(fg_span{ka, kn});
                        T->eval.push_back(v);
                        T->emeta.push_back((uint8_t)meta);
                        ++my_n;
                    }
                }
                put_row(*T, i, offsets[i], res, my_n ? begin : 0u, my_n);
            }
            cur += r;
        }
    }
    memset(out, 0, sizeof *out);
    out->n = n;
    out->n_entries = (int32_t)T->ename.size();
    out->ts = T->ts.data();
    out->meta = T->meta.data();
    out->hostname = T->host.data();
    out->appname = T->none.data();
    out->procid = T->none.data();
    out->msgid = T->none.data();
    out->msg = T->msg.data();
    out->full_msg = T->full.data();
    out->sd = T->sd.data();
    out->entry_name = T->ename.data();
    out->entry_val = T->eval.data();
    out->entry_meta = T->emeta.data();
    out->line_offsets = (const int32_t*)T;  // owner handle for emu_ltsv_free
    if (info) { info[0] = T->rounds; info[1] = T->direct; info[2] = typed && staged ? 1 : 0; }
    return 0;
}

void emu_ltsv_free(fg_batch_out* out) {
    delete (Tables*)out->line_offsets;
    memset(out, 0, sizeof *out);
}

}  // extern "C"
