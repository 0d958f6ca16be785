// emu_r3164.cpp — CPU emulation of the RFC3164 device logic (TEST INFRASTRUCTURE, see cuda_shim.h).
//
// Compiles the product's device source (fg_rfc3164.cuh: r3164_parse_line and the zone-table search) and its host-side
// zone-table builder (fg_tz.cu, which is plain C++) with g++ and replays what parse3164_kernel does with them: per CTA of
// 64 lines the contiguous byte span is copied into a 16-byte-aligned staging tile at the same in-granule offset the TMA copy
// gives it, every line that fits is parsed from the tile, the rest from the input buffer; re-joined messages go through the
// same bump allocator (with the same overflow / regrow / redo protocol the C ABI runs).  The kernel has no warp-level
// interplay — a line is parsed by one thread alone — so this replay covers the whole of its logic.
//
// Built a second time with FG_HOST_EMU_WARP (libfg_emu_warp.so): every warp of the CTA becomes 32 host threads, fg_any is a
// rendezvous of the 32 lanes (pthread barrier) and the harness checks that all lanes arrive at the same vote — same source
// line, same number of votes — which is what `__any_sync(0xFFFFFFFF, ..)` demands of r3164_parse_lockstep on the device.
#define FG_HOST_EMU 1
#include <pthread.h>

#include <algorithm>
#include <atomic>
#include <thread>
#include <cstdlib>
#include <cstring>
#include <string>
#include <vector>

#include "../../include/flowgger_cuda.h"
#include "../../flowgger_b200/csrc/fg_rfc3164.cuh"
#include "../../flowgger_b200/csrc/fg_tz.h"

namespace {
constexpr int kLines = fg::kR3164LinesPerCta;

struct Tables {
    std::vector<double> ts;
    std::vector<uint32_t> meta;
    std::vector<fg_span> host, msg, full, sd;
    std::vector<uint8_t> arena;
    int from_tile = 0, from_global = 0, redo = 0;
};

fg::TzHostTable g_tz;
std::string g_tz_dir = "\x01";

#ifdef FG_HOST_EMU_WARP
// one emulated warp: 32 lanes = 32 host threads
struct WarpState {
    pthread_barrier_t bar;
    std::atomic<uint32_t> acc[3];
    int site[3][32];
    std::atomic<int> mismatches{0};
    uint64_t votes_total = 0;
};
WarpState* g_warp = nullptr;
long long g_site_votes[4096] = {};  // rendezvous per source line of fg_rfc3164.cuh (written by lane 0 only)
thread_local int t_lane = 0;
thread_local uint64_t t_votes = 0;

// one rendezvous; site < 0 = the lane has left the walker.  Returns the OR of the predicates; *all_left = every lane has left.
bool rendezvous(bool p, int site, bool* all_left) {
    WarpState& W = *g_warp;
    const int slot = (int)(t_votes % 3);
    ++t_votes;
    if (p) W.acc[slot].fetch_or(1u);
    W.site[slot][t_lane] = site;
    pthread_barrier_wait(&W.bar);
    bool same = true, left = true;
    for (int l = 0; l < 32; ++l) {
        same = same && W.site[slot][l] == W.site[slot][0];
        left = left && W.site[slot][l] < 0;
    }
    if (!same && t_lane == 0) W.mismatches.fetch_add(1);
    const bool r = W.acc[slot].load() != 0u;
    if (t_lane == 0) {
        if (site >= 0 && site < 4096) ++g_site_votes[site];
        W.acc[(slot + 2) % 3].store(0u);  // every lane has read that slot before arriving here; nobody writes it before the next barrier
        ++W.votes_total;
    }
    if (all_left) *all_left = left;
    return r;
}
#endif
}  // namespace

#ifdef FG_HOST_EMU_WARP
namespace fg {
bool fg_emu_vote(bool p, int site) { return rendezvous(p, site, nullptr); }
void fg_emu_sync(int site) { rendezvous(false, 100000 + site, nullptr); }
}  // namespace fg
#endif

extern "C" {

// `year`: what now_utc().year() stands for.  tzdir: NULL = the system database.  arena_cap: initial capacity (small values
// exercise the regrow + redo path).  info: [5] lines parsed from the tile, from the input buffer, redo passes, (warp build) rendezvous at which the lanes
// disagreed about the vote they were at, rendezvous in total.
int emu_r3164_decode(const uint8_t* bytes, const int32_t* offsets, int32_t n, int32_t tile_bytes, int32_t strip_eol,
                     const uint8_t* invalid, int32_t year, const char* tzdir, uint32_t arena_cap, int32_t lockstep, fg_batch_out* out,
                     int32_t* info) {
    const std::string dir = tzdir ? tzdir : "";
    if (!g_tz.loaded || dir != g_tz_dir) {
        std::string err;
        if (!fg::tz_load_dir(tzdir, g_tz, err)) return -1;
        g_tz_dir = dir;
    }
    Tables* T = new Tables();
    const size_t nn = (size_t)std::max(n, 1);
    T->ts.resize(nn); T->meta.resize(nn); T->host.resize(nn); T->msg.resize(nn); T->full.resize(nn); T->sd.assign(nn, fg_span{0, 0});
    std::vector<uint8_t> tile((size_t)tile_bytes + 64);
    uint8_t* tile0 = tile.data() + ((16 - ((uintptr_t)tile.data() & 15)) & 15);  // 16-byte aligned like the shared-memory tile
    T->arena.resize(std::max<uint32_t>(arena_cap, 1));
    uint32_t counter = 0;
    long long warp_mismatches = 0, warp_votes = 0;  // FG_HOST_EMU_WARP: rendezvous at which the lanes were at different votes
    for (int attempt = 0; attempt < 2; ++attempt) {
        counter = 0;
        T->from_tile = T->from_global = 0;
        fg::R3164DeviceConfig cfg{};
        cfg.year = year;
        cfg.tz = g_tz.view();
        cfg.arena = T->arena.data();
        cfg.arena_cap = (uint32_t)T->arena.size();
        cfg.arena_counter = &counter;
        for (int first = 0; first < n; first += kLines) {
            const int last = std::min(n, first + kLines);
            const int base = fg::span_base(offsets[first]);
            int r = 0;
            while (first + r < last && offsets[first + r + 1] - base <= tile_bytes) ++r;
            if (r > 0) {
                const uint32_t nbytes = fg::span_copy_bytes(base, offsets[first + r]);
                // the device buffer is padded; here only the bytes that exist are copied, the rest of the granule is zero
                const int64_t avail = (int64_t)offsets[n] - base;
                memset(tile0, 0, nbytes);
                memcpy(tile0, bytes + base, (size_t)std::min<int64_t>(nbytes, avail));
            }
            auto parse_one = [&](int i) {  // what one thread of the CTA does (fg_parse3164.cu)
                const bool have = i < last;
                const int o0 = have ? offsets[i] : 0, o1 = have ? offsets[i + 1] : 0;
                const bool fits = have && i - first < r;
                const uint8_t* lp = fits ? tile0 + (o0 - base) : bytes + o0;
                int len = o1 - o0;
                bool bad = false;
                if (have && strip_eol && len > 0) {
                    len = fg::strip_terminator(lp, 0, len, strip_eol);
                    bad = invalid != nullptr && invalid[i] != 0;
                }
                fg::R3Out res;
                if (lockstep) {  // the walker the kernel is built with (FG_R3_LOCKSTEP = 1); every lane of the warp calls it
                    fg::r3164_parse_lockstep(lp, len, have && !bad, cfg, res);
                    if (bad) res.status = FG_ES_INVALID_UTF8;
                } else if (bad || !have) {
                    res.status = FG_ES_INVALID_UTF8;
                    res.facility = res.severity = 0xFFu;
                    res.flags = 0u;
                    res.ts = 0.0;
                } else {
                    fg::r3164_parse_line(lp, len, cfg, res);
                }
                if (!have) return;
                const bool ok = res.status == FG_ST_OK;
                T->ts[i] = ok ? res.ts : 0.0;
                T->meta[i] = res.status | (res.facility << 8) | (res.severity << 16) | (res.flags << 24);
                T->host[i] = ok ? fg_span{o0 + res.host_o, res.host_l} : fg_span{-1, 0};
                T->msg[i] = ok ? fg_span{(res.flags & fg::kR3FlagMsgArena) ? res.msg_o : o0 + res.msg_o, res.msg_l} : fg_span{-1, 0};
                T->full[i] = ok ? fg_span{o0, res.full_l} : fg_span{-1, 0};
            };
#ifdef FG_HOST_EMU_WARP
            for (int w0 = first; w0 < first + kLines && w0 < last; w0 += 32) {  // the warps of the CTA that hold lines
                WarpState W;
                pthread_barrier_init(&W.bar, nullptr, 32);
                for (auto& a : W.acc) a.store(0u);
                g_warp = &W;
                std::thread lanes[32];
                for (int l = 0; l < 32; ++l)
                    lanes[l] = std::thread([&, l] {
                        t_lane = l;
                        t_votes = 0;
                        parse_one(w0 + l);
                        bool all_left = false;  // keep meeting the other lanes until every one of them has left the walker
                        while (!all_left) rendezvous(false, -1, &all_left);
                    });
                for (auto& th : lanes) th.join();
                pthread_barrier_destroy(&W.bar);
                warp_mismatches += W.mismatches.load();
                warp_votes += (long long)W.votes_total;
                g_warp = nullptr;
            }
            T->from_tile += std::min(r, last - first);
            T->from_global += (last - first) - std::min(r, last - first);
#else
            for (int i = first; i < last; ++i) {
                parse_one(i);
                (i - first < r ? T->from_tile : T->from_global)++;
            }
#endif
        }
        if (counter <= T->arena.size()) break;
        T->arena.assign((size_t)counter + counter / 8 + 1024, 0);  // regrow_tables, then the batch is redone
        ++T->redo;
    }
    memset(out, 0, sizeof *out);
    out->n = n;
    out->ts = T->ts.data();
    out->meta = T->meta.data();
    out->hostname = T->host.data();
    out->msg = T->msg.data();
    out->full_msg = T->full.data();
    out->sd = T->sd.data();
    out->arena = T->arena.data();
    out->arena_bytes = (int64_t)counter;
    out->line_offsets = (const int32_t*)T;  // owner handle for emu_r3164_free
    if (info) { info[0] = T->from_tile; info[1] = T->from_global; info[2] = T->redo; info[3] = (int32_t)warp_mismatches; info[4] = (int32_t)std::min<long long>(warp_votes, 0x7FFFFFFF); }
    return 0;
}

#ifdef FG_HOST_EMU_WARP
// votes per source line of fg_rfc3164.cuh since the last call (a lock-step iteration count per loop: the walker's cost model)
int emu_r3164_site_votes(int32_t* lines, int64_t* counts, int cap) {
    int k = 0;
    for (int l = 0; l < 4096 && k < cap; ++l)
        if (g_site_votes[l]) {
            lines[k] = l;
            counts[k] = g_site_votes[l];
            g_site_votes[l] = 0;
            ++k;
        }
    return k;
}
#endif

void emu_r3164_free(fg_batch_out* out) {
    delete (Tables*)out->line_offsets;
    memset(out, 0, sizeof *out);
}

// the packed zone table as the kernel searches it: 1 + offset stored, or 0 when `name` is no identifier
int emu_tz_lookup(const char* tzdir, const char* name, int64_t local, int32_t* offset) {
    const std::string dir = tzdir ? tzdir : "";
    if (!g_tz.loaded || dir != g_tz_dir) {
        std::string err;
        if (!fg::tz_load_dir(tzdir, g_tz, err)) return -1;
        g_tz_dir = dir;
    }
    const fg::TzDeviceTable V = g_tz.view();
    const int z = fg::tz_find(V, (const uint8_t*)name, 0, (int)strlen(name));
    if (z < 0) return 0;
    *offset = fg::tz_offset_local(V, z, (long long)local);
    return 1;
}
int emu_tz_count(const char* tzdir) {
    int32_t o;
    if (emu_tz_lookup(tzdir, "UTC", 0, &o) < 0) return -1;
    return g_tz.n_names();
}

}  // extern "C"
