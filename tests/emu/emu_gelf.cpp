// emu_gelf.cpp — CPU emulation of the GELF device logic (TEST INFRASTRUCTURE, see cuda_shim.h).
//
// Compiles the product's device sources (fg_gelffast.cuh: stage-1 bitmaps, line pass, gf_member, gf_finish; fg_gelf.cuh: the
// exact parser and phase 2) with g++ and replays what parse_gelf_kernel / post_gelf_kernel do with them — CTA rounds over
// a staging tile, slot reservation, staged rows, the slow list — one lane at a time.  The result has the layout of
// fg_batch_out (columnar rows + side table), so the CPU test-suite can push it through the product's materialiser and
// compare with the oracle without a GPU.
#define FG_HOST_EMU 1
#include <algorithm>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>

#include "../../include/flowgger_cuda.h"
#include "../../flowgger_b200/csrc/fg_gelffast.cuh"

namespace {
constexpr int kLines = fg::kGelfLinesPerCta;
constexpr int kSlots = fg::kGelfStageSlots;

struct Tables {
    std::vector<double> ts;
    std::vector<uint32_t> meta;
    std::vector<fg_span> host, msg, full, sd, none;
    std::vector<fg_span> ename;
    std::vector<uint64_t> eval;
    std::vector<uint8_t> emeta;
    int rounds = 0, slow = 0, bound_violations = 0;
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

void init_pow10() {
    static bool done = false;
    if (done) return;
    for (int k = 0; k <= 308; ++k) {
        char buf[16];
        snprintf(buf, sizeof buf, "1e%d", k);
        fg::g_pow10.v[k] = strtod(buf, nullptr);
    }
    done = true;
}
}  // namespace

extern "C" {

// out[4]: the Q / B / P masks of a 16-byte granule and its control-byte flag (0 / 1)
void emu_gelf_bits16(const uint8_t* p, uint32_t* out) {
    uint32_t w[4], c;
    memcpy(w, p, 16);
    fg::gf_bits16(w[0], w[1], w[2], w[3], out[0], out[1], out[2], c);
    out[3] = c != 0u;
}

int emu_gelf_decode(const uint8_t* bytes, const int32_t* offsets, int32_t n, int32_t tile_bytes, int32_t strip_eol,
                    const uint8_t* invalid, fg_batch_out* out, int32_t* info /* [3]: rounds, slow-path lines, slot-bound violations */) {
    init_pow10();
    Tables* T = new Tables();
    const size_t nn = (size_t)std::max(n, 1);
    T->ts.resize(nn); T->meta.resize(nn); T->host.resize(nn); T->msg.resize(nn); T->full.resize(nn); T->sd.resize(nn);
    T->none.assign(nn, fg_span{-1, 0});
    const int64_t total_bytes = n > 0 ? offsets[n] : 0;
    std::vector<uint8_t> tile((size_t)tile_bytes + 64);
    std::vector<uint32_t> bmQ((size_t)tile_bytes / 32 + 8), bmB(bmQ.size()), bmP(bmQ.size()), anyK(bmQ.size() / 32 + 8);
    std::vector<fg_span> st_name((size_t)kSlots + fg::kMaxLocalMembers);
    std::vector<uint64_t> st_val(st_name.size());
    std::vector<uint8_t> st_meta(st_name.size());
    std::vector<uint32_t> slow_list;

    for (int first = 0; first < n; first += kLines) {
        const int last = std::min(n, first + kLines);
        int cur = first;
        while (cur < last) {
            const int base = fg::span_base(offsets[cur]);
            int r = 0;
            while (cur + r < last && offsets[cur + r + 1] - base <= tile_bytes) ++r;
            if (r == 0) {
                slow_list.push_back((uint32_t)cur);
                ++cur;
                continue;
            }
            ++T->rounds;
            const uint32_t nbytes = fg::span_copy_bytes(base, offsets[cur + r]);
            for (uint32_t k = 0; k < nbytes; ++k) tile[k] = (int64_t)base + k < total_bytes ? bytes[base + k] : 0;  // the bulk copy
            const int nword = (int)((nbytes + 31u) >> 5);
            std::fill(anyK.begin(), anyK.end(), 0u);
            for (int g = 0; g < nword; ++g) {
                uint32_t lo[4], hi[4] = {0, 0, 0, 0};
                emu_gelf_bits16(tile.data() + 32 * g, lo);
                if ((uint32_t)(32 * g + 16) < nbytes) emu_gelf_bits16(tile.data() + 32 * g + 16, hi);
                bmQ[g] = lo[0] | (hi[0] << 16);
                bmB[g] = lo[1] | (hi[1] << 16);
                bmP[g] = lo[2] | (hi[2] << 16);
                if (lo[3] | hi[3]) anyK[g >> 5] |= 1u << (g & 31);
            }
            for (int k = 0; k < 4; ++k) bmQ[nword + k] = bmB[nword + k] = bmP[nword + k] = 0;
            uint32_t run = 0;
            int done = 0;
            for (int tid = 0; tid < r; ++tid) {
                const int i = cur + tid, o0 = offsets[i];
                const int ls = o0 - base;
                int le = offsets[i + 1] - base;
                bool bad = false;
                if (strip_eol && le > ls) {
                    le = fg::strip_terminator(tile.data(), ls, le, strip_eol);
                    if (invalid && invalid[i]) bad = true;
                }
                const bool walk = !bad;
                uint16_t cuts[fg::kMaxLocalMembers];
                int open = 0, m = -1;
                if (walk && !fg::gf_has_ctrl(tile.data(), anyK.data(), ls, le))
                    m = fg::gf_line_members(tile.data(), bmQ.data(), bmB.data(), bmP.data(), ls, le, cuts, fg::kMaxLocalMembers, open, true);
                bool regular = m >= 0;
                const uint32_t nb = (walk && regular) ? (uint32_t)m : 0u;
                if (run + nb > (uint32_t)kSlots) break;  // the round is cut here; the rest is redone
                const uint32_t slot0 = run;
                run += nb;
                ++done;
                // (4) one member at a time: validation + conversion; numbers in a second pass
                fg::Members M;
                M.m = 0;
                M.spilled = false;
                uint32_t n_plain = 0;
                for (uint32_t k = 0; k < nb && regular; ++k) {
                    int2 name = make_int2(0, 0);
                    unsigned long long val = 0;
                    uint32_t meta = 0;
                    const int a = k == 0 ? open + 1 : (int)cuts[k - 1] + 1;
                    if (!fg::gf_member(tile.data(), bmQ.data(), bmB.data(), a, (int)cuts[k], o0, ls, true, name, val, meta) ||
                        (meta == fg::kGfNumber && !fg::gf_member_number(tile.data(), val, val, meta))) {
                        regular = false;
                        break;
                    }
                    M.name[k] = name;
                    M.val[k] = val;
                    M.meta[k] = (uint8_t)meta;
                    M.m = k + 1;
                    if ((meta >> 5) == (uint32_t)fg::GKEY_OTHER) ++n_plain;
                }
                if (walk && !regular) {
                    slow_list.push_back((uint32_t)i);
                    continue;
                }
                fg::LineResult res;
                fg::gelf_result_init(res);
                if (walk) {
                    fg::GelfAcc g;
                    g.status = FG_ST_OK; g.flags = 0; g.kept = 0; g.have_ts = false;
                    fg::EntrySink stage = {(int2*)st_name.data(), (unsigned long long*)st_val.data(), st_meta.data()};
                    fg::gf_finish(tile.data() + ls, o0, M, res, g, stage, slot0);
                    if (g.kept > n_plain || g.kept > nb) ++T->bound_violations;
                    fg::gelf_finalize(res, g);
                }
                if (bad) { res.status = FG_ES_INVALID_UTF8; res.n_entries = 0; res.full_o = 0; }
                const uint32_t my_n = (walk && res.status == FG_ST_OK) ? res.n_entries : 0u;
                const uint32_t begin = my_n ? (uint32_t)T->ename.size() : 0u;
                for (uint32_t k = 0; k < my_n; ++k) {
                    T->ename.push_back(st_name[slot0 + k]);
                    T->eval.push_back(st_val[slot0 + k]);
                    T->emeta.push_back(st_meta[slot0 + k]);
                }
                put_row(*T, i, o0, res, begin, my_n);
            }
            cur += done;
        }
    }
    // post_gelf_kernel
    std::vector<fg_span> tname;
    std::vector<uint64_t> tval;
    std::vector<uint8_t> tmeta;
    for (uint32_t line : slow_list) {
        ++T->slow;
        const int o0 = offsets[line];
        int len = offsets[line + 1] - o0;
        len = fg::strip_terminator(bytes, o0, o0 + len, strip_eol) - o0;
        tname.assign((size_t)len / 3 + 64, fg_span{0, 0});
        tval.assign(tname.size(), 0);
        tmeta.assign(tname.size(), 0);
        fg::EntrySink tmp = {(int2*)tname.data(), (unsigned long long*)tval.data(), tmeta.data()};
        fg::LineResult res;
        fg::gelf_parse_line(bytes + o0, len, o0, 0u, true, res, tmp);
        const uint32_t my_n = res.status == FG_ST_OK ? res.n_entries : 0u;
        const uint32_t begin = my_n ? (uint32_t)T->ename.size() : 0u;
        for (uint32_t k = 0; k < my_n; ++k) {
            T->ename.push_back(tname[k]);
            T->eval.push_back(tval[k]);
            T->emeta.push_back(tmeta[k]);
        }
        put_row(*T, (int)line, o0, res, begin, my_n);
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
    out->line_offsets = (const int32_t*)T;  // owner handle for emu_gelf_free
    if (info) { info[0] = T->rounds; info[1] = T->slow; info[2] = T->bound_violations; }
    return 0;
}

void emu_gelf_free(fg_batch_out* out) {
    delete (Tables*)out->line_offsets;
    memset(out, 0, sizeof *out);
}

}  // extern "C"
