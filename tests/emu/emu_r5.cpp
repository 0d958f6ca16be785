// emu_r5.cpp — CPU emulation of the RFC5424 device logic (TEST INFRASTRUCTURE, see cuda_shim.h).
//
// Compiles the product's walker sources (fg_r5fast.cuh: stage-1 classification, stage-2 bit-walk, unescape;
// fg_rfc5424.cuh: the wide-path scanner) with g++ and replays what parse5424_kernel and post5424_kernel (unescape_lines,
// wide_lines) do with them — CTA rounds over a staging tile, rows staged in the line's own bytes, side-table
// placement, work lists — one lane at a time.  The result has the exact layout of fg_batch_out, so the CPU test-suite
// can push it through the product's materialiser and compare with the oracle without a GPU.  It is built into
// tests/emu/libfg_emu.so by tests/emu/build.py and loaded by tests only.
#define FG_HOST_EMU 1
#include <algorithm>
#include <cstdlib>
#include <cstring>
#include <vector>

#include "../../include/flowgger_cuda.h"
#include "../../flowgger_b200/csrc/fg_r5fast.cuh"
#include "../../flowgger_b200/csrc/fg_rfc5424.cuh"
#include "../../flowgger_b200/csrc/fg_dtoa.cuh"

namespace {
constexpr int kLines = fg::kRfc5424LinesPerCta;

struct Tables {
    std::vector<fg_row5424> rows;
    std::vector<uint64_t> e8;
    std::vector<uint8_t> arena;
    std::vector<fg_wide_row> wide;
    std::vector<fg_span> wname;
    std::vector<uint64_t> wval;
    std::vector<uint8_t> wmeta;
    std::vector<uint32_t> esc_list, wide_list;
};

void put_row(Tables& t, int i, const fg::R5Fast& r, uint32_t first, uint32_t n) {
    fg_row5424 row;
    memset(&row, 0, sizeof row);
    row.meta = r.status == FG_ST_OK ? (r.facility << 8) | (r.severity << 16) | (r.flags << 24) : r.status | 0x00FFFF00u;
    row.sd_first = first;
    if (r.status == FG_ST_OK) {
        row.ts = r.ts;
        row.sd_count = (uint16_t)n;
        row.sp[0] = (uint16_t)r.sp1; row.sp[1] = (uint16_t)r.sp2; row.sp[2] = (uint16_t)r.sp3;
        row.sp[3] = (uint16_t)r.sp4; row.sp[4] = (uint16_t)r.sp5;
        row.msg_off = (uint16_t)r.msg_o;
        row.msg_len = (uint16_t)r.msg_l;
    }
    t.rows[(size_t)i] = row;
}
}  // namespace

extern "C" {

// 16-byte classification of stage 1, exposed so tests can pin the SWAR identities against a per-byte definition
uint32_t emu5424_classify16(const uint8_t* p) {
    uint32_t w[4];
    memcpy(w, p, 16);
    return fg::r5_classify16(w[0], w[1], w[2], w[3]);
}
// f64 -> text of the GELF encoder (fg_dtoa.cuh), for the CPU tests of the Grisu2 restatement
int emu_json_f64(double v, uint8_t* out) { return fg::json_f64(v, out); }

int emu5424_decode(const uint8_t* bytes, const int32_t* offsets, int32_t n, int32_t tile_bytes, int32_t strip_eol,
                   const uint8_t* invalid, fg_batch_out* out) {
    Tables* T = new Tables();
    T->rows.resize((size_t)std::max(n, 1));
    const int64_t total_bytes = n > 0 ? offsets[n] : 0;
    std::vector<uint8_t> tile((size_t)tile_bytes + 64);
    std::vector<uint32_t> bmI((size_t)tile_bytes / 32 + 8);
    for (int first = 0; first < n; first += kLines) {
        const int last = std::min(n, first + kLines);
        int cur = first;
        while (cur < last) {
            const int base = fg::span_base(offsets[cur]);
            int r = 0;
            while (cur + r < last && offsets[cur + r + 1] - base <= tile_bytes) ++r;
            if (r == 0) {
                T->wide_list.push_back((uint32_t)cur);
                ++cur;
                continue;
            }
            const uint32_t nbytes = fg::span_copy_bytes(base, offsets[cur + r]);
            for (uint32_t k = 0; k < nbytes; ++k) tile[k] = (int64_t)base + k < total_bytes ? bytes[base + k] : 0;  // the bulk copy
            uint16_t* bmI16 = (uint16_t*)bmI.data();
            const int ngran = (int)(nbytes >> 4);
            for (int g = 0; g < ngran; ++g) bmI16[g] = (uint16_t)emu5424_classify16(tile.data() + 16 * g);
            for (int k = 0; k < 6; ++k) bmI16[ngran + k] = 0;
            for (int tid = 0; tid < r; ++tid) {
                const int i = cur + tid;
                const int ls = offsets[i] - base;
                int le = offsets[i + 1] - base;
                bool bad = false;
                if (strip_eol && le > ls) {
                    le = fg::strip_terminator(tile.data(), ls, le, strip_eol);
                    if (invalid && invalid[i]) bad = true;
                }
                const bool too_long = le - ls > 65535;
                fg::R5Fast res;
                const bool regular = fg::r5_regular(tile.data(), bmI.data(), ls, (too_long || bad) ? ls : le, res);
                if (bad) {
                    res.status = FG_ES_INVALID_UTF8;
                    res.n_entries = 0;
                }
                if (!regular && !bad) {
                    T->wide_list.push_back((uint32_t)i);
                    continue;
                }
                const uint32_t my_n = res.status == FG_ST_OK ? res.n_entries : 0u;
                const uint32_t first_e = my_n ? (uint32_t)T->e8.size() : 0u;
                for (uint32_t k = 0; k < my_n; ++k) T->e8.push_back(res.stage[k]);
                if (my_n && res.esc) T->esc_list.push_back((uint32_t)i);
                put_row(*T, i, res, first_e, my_n);
            }
            cur += r;
        }
    }
    // post5424_kernel, unescape_lines: arena records are [u16 length][bytes], 2-byte aligned
    for (uint32_t line : T->esc_list) {
        const fg_row5424& row = T->rows[line];
        const int o0 = offsets[line];
        for (uint32_t e = row.sd_first; e < row.sd_first + row.sd_count; ++e) {
            const uint64_t v = T->e8[e];
            if (!(v & fg::kE8Header) && (v & fg::kE8Esc)) {
                const int ne = (int)FG_E8_B(v), ve = (int)FG_E8_C(v);
                const size_t at = T->arena.size();
                T->arena.resize(at + ((2 + (size_t)(ve - (ne + 2)) + 1) & ~(size_t)1));  // reserved from the raw length
                const uint16_t l16 = (uint16_t)fg::r5_unescape_to(bytes + o0 + ne + 2, ve - (ne + 2), T->arena.data() + at + 2);
                memcpy(T->arena.data() + at, &l16, 2);
                T->e8[e] = (v & 0xFFFFFFFFull) | ((uint64_t)(at >> 1) << 32) | fg::kE8Arena;
            }
        }
    }
    // post5424_kernel, wide_lines
    for (uint32_t line : T->wide_list) {
        const int o0 = offsets[line];
        int len = offsets[line + 1] - o0;
        bool bad = false;
        if (strip_eol && len > 0) {
            len = fg::strip_terminator(bytes, o0, o0 + len, strip_eol) - o0;
            if (invalid && invalid[line]) bad = true;
        }
        if (bad) len = 0;
        int marks[6][32];
        fg::LineResult res, again;
        fg::EntrySink none = {nullptr, nullptr, nullptr};
        fg::rfc5424_parse_line<32>(bytes + o0, len, o0, &marks[0][0], res, none, 0u, false);
        const uint32_t cnt = (!bad && res.status == FG_ST_OK) ? res.n_entries : 0u;
        const uint32_t wbase = (uint32_t)T->wname.size();
        T->wname.resize(wbase + cnt);
        T->wval.resize(wbase + cnt);
        T->wmeta.resize(wbase + cnt);
        fg::EntrySink sink = {(int2*)T->wname.data(), (unsigned long long*)T->wval.data(), T->wmeta.data()};
        if (cnt) fg::rfc5424_parse_line<32>(bytes + o0, len, o0, &marks[0][0], again, sink, wbase, true);
        for (uint32_t k = 0; k < cnt; ++k) {
            const uint32_t e = wbase + k;
            const uint8_t m = T->wmeta[e];
            if ((m & 0x07u) == 0u && (m & 0x08u)) {
                const uint64_t v = T->wval[e];
                const uint32_t off = (uint32_t)v, l = (uint32_t)(v >> 32);
                const uint32_t ul = (uint32_t)fg::r5_unescape(bytes + off, (int)l, nullptr);
                const size_t at = T->arena.size();
                T->arena.resize(at + ul + 2);
                fg::r5_unescape(bytes + off, (int)l, T->arena.data() + at);
                T->arena.resize(at + ((ul + 1) & ~(size_t)1));
                T->wval[e] = (uint64_t)at | ((uint64_t)ul << 32);
                T->wmeta[e] = 0x80u;
            }
        }
        if (bad) {
            res.status = FG_ES_INVALID_UTF8;
            res.flags = 0;
            res.facility = res.severity = 0xFFu;
        }
        const bool ok = res.status == FG_ST_OK;
        if (!ok) {
            fg_row5424 row;
            memset(&row, 0, sizeof row);
            row.meta = res.status | 0x00FFFF00u;
            T->rows[line] = row;
            continue;
        }
        fg_wide_row w;
        memset(&w, 0, sizeof w);
        w.line = (int32_t)line;
        w.meta = res.status | (res.facility << 8) | (res.severity << 16) | ((res.flags | fg::kFlagWide) << 24);
        w.ts = res.ts;
        w.hostname = fg_span{ok ? o0 + res.host_o : -1, res.host_l};
        w.appname = fg_span{ok ? o0 + res.app_o : -1, res.app_l};
        w.procid = fg_span{ok ? o0 + res.proc_o : -1, res.proc_l};
        w.msgid = fg_span{ok ? o0 + res.mid_o : -1, res.mid_l};
        w.msg = fg_span{ok && res.msg_o >= 0 ? o0 + res.msg_o : -1, res.msg_l};
        w.full_msg = fg_span{ok && res.full_o >= 0 ? o0 + res.full_o : -1, res.full_l};
        w.sd = fg_span{(int32_t)wbase, (int32_t)(ok ? cnt : 0u)};
        fg_row5424 row;
        memset(&row, 0, sizeof row);
        row.ts = res.ts;
        row.meta = w.meta;
        row.sd_first = (uint32_t)T->wide.size();
        T->rows[line] = row;
        T->wide.push_back(w);
    }
    memset(out, 0, sizeof *out);
    out->n = n;
    out->n_entries = (int32_t)T->wname.size();
    out->entry_name = T->wname.data();
    out->entry_val = T->wval.data();
    out->entry_meta = T->wmeta.data();
    out->rows5424 = T->rows.data();
    out->entries8 = T->e8.data();
    out->n_entries8 = (int32_t)T->e8.size();
    out->n_wide = (int32_t)T->wide.size();
    out->wide_rows = T->wide.data();
    out->arena = T->arena.data();
    out->arena_bytes = (int64_t)T->arena.size();
    out->line_offsets = (const int32_t*)T;  // owner handle for emu5424_free (tests never read line_offsets of an emu result)
    return 0;
}

void emu5424_free(fg_batch_out* out) {
    delete (Tables*)out->line_offsets;
    memset(out, 0, sizeof *out);
}

}  // extern "C"
