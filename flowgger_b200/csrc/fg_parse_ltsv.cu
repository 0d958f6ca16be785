// fg_parse_ltsv.cu — the LTSV decoder on sm_90a: bytes -> row columns + side table, on the bitmap pipeline, part-parallel.
//
//   parse_ltsv_kernel   one CTA = 64 consecutive lines, 256 threads.  Per round:
//     (1) thread 0 issues ONE TMA bulk copy (cp.async.bulk, SASS UBLKCP) of the lines' contiguous byte span into the
//         shared-memory tile — HBM is read once, coalesced, with no per-thread global loads;
//     (2) all threads sweep the tile 32 bytes per step into the TAB bitmap (fg_ltsvfast.cuh stage 1);
//     (3) one thread per line counts its TABs; a CTA scan reserves one SLOT per part; the thread lists the TAB positions
//         into its slots;
//     (4) one thread per SLOT (all 256 threads, over all slots of the round) classifies its part: packed side-table row
//         into the slot, or — for the reserved keys — the slot number into the line's record (shared-memory atomics);
//     (5) one thread per typed row parses the schema value; one thread per line parses `time` / `level` and settles the
//         line's status (the first failing part wins);
//     (6) the rows of the lines that decoded are compacted by two ballot scans over the slots, placed by ONE global atomic
//         and written as three coalesced columns; then the row columns of the lines.
//   Lines with a repeated `time` / `level` key, lines that do not fit the tile and lines with more parts than the CTA has
//   slots are parsed by the round-1 scanner (fg_ltsv.cuh) straight from global memory, through the scratch table.
#include "fg_kernels.cuh"

#include "fg_common.cuh"
#include "fg_ltsvfast.cuh"
#include "fg_status.h"
#include "fg_tma.cuh"

namespace fg {

namespace {

constexpr int kLines = kLtsvLinesPerCta;
constexpr int kThreads = kLtsvThreadsPerCta;
constexpr int kWarps = kThreads / 32;
static_assert(kThreads >= kLines && kWarps >= 2, "the line phases need one thread per line");
constexpr int kLtsvCtasPerSm = 4;  // shared memory (tile ~28 KB + slots) allows 4 CTAs: 64 registers keep all of them resident
constexpr int kStageSlots = kLtsvStageSlots;
constexpr int kSchemaKeys = 64, kSchemaBlob = 1024, kSuffixBlob = 64;  // larger schemas are read from global memory

__device__ __forceinline__ void write_row(const ParseParams& P, int i, int o0, const LineResult& res, uint32_t my_begin, uint32_t my_n) {
    const bool ok = res.status == FG_ST_OK;
    P.ts[i] = res.ts;
    P.meta[i] = res.status | (res.facility << 8) | (res.severity << 16) | (res.flags << 24);
    P.host[i] = make_int2(res.host_o >= 0 ? o0 + res.host_o : -1, res.host_l);
    P.msg[i] = make_int2(res.msg_o >= 0 ? o0 + res.msg_o : -1, res.msg_l);
    // error rows: full.off = absolute byte offset of the failing part (LTSV side effects), len 0
    P.full[i] = ok ? make_int2(res.full_o >= 0 ? o0 + res.full_o : -1, res.full_l) : make_int2(o0 + max(res.full_o, 0), 0);
    P.sd[i] = make_int2((int)my_begin, (int)my_n);
}

// one line through the round-1 scanner, straight from global memory (all threads call; thread 0 does the work)
__device__ __forceinline__ void direct_line(const ParseParams& P, int line, const EntrySink& sink, const EntrySink& tmp) {
    const bool act = threadIdx.x == 0;
    const int d0 = __ldg(P.offsets + line);
    int len = act ? __ldg(P.offsets + line + 1) - d0 : 0;
    bool bad_utf8 = false;
    if (act && P.strip_eol && len > 0) {
        len = strip_terminator(P.bytes + d0, 0, len, P.strip_eol);
        if (P.line_invalid != nullptr && P.line_invalid[line]) {
            bad_utf8 = true;
            len = 0;
        }
    }
    LineResult res;
    const uint32_t sidx = (uint32_t)d0 / 2u + (uint32_t)(P.line0 + line);  // a row needs >= 1 input byte + its TAB
    ltsv_parse_line(P.bytes + d0, len, d0, sidx, act, P.ltsv, res, tmp);
    if (bad_utf8) {
        res.status = FG_ES_INVALID_UTF8;
        res.n_entries = 0;
        res.full_o = 0;
    }
    if (act) {
        const uint32_t my_n = res.status == FG_ST_OK ? res.n_entries : 0u;
        uint32_t my_begin = 0;
        if (my_n) {
            const uint32_t eb = atomicAdd(P.entry_counter, my_n);
            if ((unsigned long long)eb + my_n <= (unsigned long long)P.entry_cap) {
                my_begin = eb;
                for (uint32_t k = 0; k < my_n; ++k) {
                    sink.name[eb + k] = tmp.name[sidx + k];
                    sink.val[eb + k] = tmp.val[sidx + k];
                    sink.meta[eb + k] = tmp.meta[sidx + k];
                }
            }
        }
        write_row(P, line, d0, res, my_begin, my_n);
    }
}

// per-line record of a round (shared memory, one array per field)
struct LineRecs {
    int ls[kLines];
    uint32_t slot0[kLines], nb[kLines];                                       // the line's slots
    uint32_t host_s[kLines], msg_s[kLines], time_s[kLines], level_s[kLines];  // 1 + slot of the LAST such part (0: none)
    uint32_t dups[kLines];       // #time | #level << 8
    uint32_t flags[kLines];      // FG_FLAG_MISSING_VALUE
    uint32_t err[kLines];        // min over failed typed values of (part index << 8 | status)
    uint32_t dense0[kLines];     // rows of the round before the line's first one
    uint32_t state[kLines];      // 0: decoded, rows kept; 1: direct path; 2: not in this round; 3: decoded, no rows (error)
    int t_a[kLines], t_b[kLines];  // value of the `time` part
    double ts[kLines];
    uint32_t ts_ok[kLines];
    uint32_t tlist[4][kLines];   // lines by lt_time_class
    uint32_t tcount[4];
    uint32_t rowmask[kLtsvStageSlots / 32];  // bit s: slot s holds a row
    uint32_t ycount[5], ybase[5], ypos[5];   // TYPED: typed rows per fg_ltsv_type (counting sort of the slots by type)
};

template <bool TYPED>
__global__ void __launch_bounds__(kThreads, kLtsvCtasPerSm) parse_ltsv_kernel(const __grid_constant__ ParseParams P) {
    extern __shared__ __align__(128) uint8_t tile[];
    __shared__ __align__(8) uint64_t mbar;
    __shared__ uint32_t scan_ws[33];
    __shared__ uint32_t s_ebase, s_slots, s_direct;
    __shared__ LineRecs L;
    // TYPED: the CTA's copy of the schema and the suffixes (a few hundred bytes)
    __shared__ uint8_t s_names[TYPED ? kSchemaBlob : 4];
    __shared__ int32_t s_name_off[TYPED ? kSchemaKeys + 1 : 1];
    __shared__ int32_t s_types[TYPED ? kSchemaKeys : 1];
    __shared__ uint8_t s_suffix[TYPED ? kSuffixBlob : 4];
    __shared__ uint32_t s_first[8];
    __shared__ uint32_t s_len_mask;

    const int tid = threadIdx.x;
    const uint32_t lane = (uint32_t)tid & 31u, wid = (uint32_t)tid >> 5;
    const int first = blockIdx.x * kLines;
    const int last = min(P.n, first + kLines);
    // behind the tile: the TAB bitmap (tile_bytes / 32 + 4 words), the slots (row | typed value | TAB position | line)
    const int bm_words = P.tile_bytes / 32 + 4;
    uint32_t* bmT = reinterpret_cast<uint32_t*>(tile + P.tile_bytes);
    unsigned long long* stage = reinterpret_cast<unsigned long long*>(bmT + bm_words);
    unsigned long long* stage_val = stage + kStageSlots;  // TYPED only
    uint16_t* tabs = reinterpret_cast<uint16_t*>(stage + (TYPED ? 2 : 1) * kStageSlots);
    uint16_t* ylist = tabs + kStageSlots;  // TYPED only: the typed rows' slots, grouped by type
    uint8_t* slot_line = reinterpret_cast<uint8_t*>(ylist + (TYPED ? kStageSlots : 0));
    if (*P.bad_offsets) return;  // CTA-uniform
    TileStage tstage = {&mbar};
    tstage.init();
    LtsvDeviceConfig cfg = P.ltsv;
    LtsvSchemaView S = {cfg.names, cfg.name_off, cfg.types, cfg.n_schema, 0xFFFFFFFFu, nullptr};
    if (TYPED) {
        const int nblob = cfg.n_schema > 0 ? cfg.name_off[cfg.n_schema] : 0, nsuf = cfg.suffix_off[5];
        if (cfg.n_schema <= kSchemaKeys && nblob <= kSchemaBlob && nsuf <= kSuffixBlob) {  // CTA-uniform
            for (int k = tid; k < nblob; k += kThreads) s_names[k] = cfg.names[k];
            for (int k = tid; k <= cfg.n_schema; k += kThreads) s_name_off[k] = cfg.name_off[k];
            for (int k = tid; k < cfg.n_schema; k += kThreads) s_types[k] = cfg.types[k];
            for (int k = tid; k < nsuf; k += kThreads) s_suffix[k] = cfg.suffix[k];
            __syncthreads();
            if (tid == 0) {
                uint32_t lm;
                lt_schema_filters(s_names, s_name_off, cfg.n_schema, lm, s_first);
                s_len_mask = lm;
            }
            __syncthreads();
            cfg.suffix = s_suffix;
            S = LtsvSchemaView{s_names, s_name_off, s_types, cfg.n_schema, s_len_mask, s_first};
        }
    }
    __syncthreads();

    const EntrySink sink = {P.entry_name, P.entry_val, P.entry_meta};
    const EntrySink tmp = {P.tmp_name, P.tmp_val, P.tmp_meta};
    int cur = first;
    bool direct_next = false;  // CTA-uniform: line `cur` must take the direct path (more parts than the CTA has slots)
    while (cur < last) {
        // ---- the lines of this round ------------------------------------------------------------------------------
        const bool lt = tid < kLines;  // line threads
        const int i = cur + tid;
        // tile_bytes <= 65024 (launch_parse_ltsv): a line inside the tile is shorter than 64 KiB, positions fit 16 bits
        // (a direct_next round has no tile — no line fits -1 bytes — so r == 0 sends line `cur` down the direct path)
        const TileRound t = plan_round(P.offsets, cur, last, direct_next ? -1 : P.tile_bytes, lt);
        const int o0 = t.o0, o1 = t.o1, base = t.base;
        int r = t.r;
        if (r == 0) {
            direct_next = false;
            direct_line(P, cur, sink, tmp);
            __syncthreads();
            cur += 1;
            continue;
        }
        const uint32_t nbytes = span_copy_bytes(base, __ldg(P.offsets + cur + r));
        tstage.load(tile, P.bytes + base, nbytes);

        // ---- (2) the TAB bitmap of the whole tile, 32 bytes (= one word) per thread per step --------------------------
        const int nword = (int)((nbytes + 31u) >> 5);  // the tile allocation is a multiple of 512 bytes: reading the odd granule is safe
        for (int g = tid; g < nword; g += kThreads) {
            const uint4 v0 = reinterpret_cast<const uint4*>(tile)[2 * g], v1 = reinterpret_cast<const uint4*>(tile)[2 * g + 1];
            bmT[g] = lt_tab16(v0.x, v0.y, v0.z, v0.w) | (lt_tab16(v1.x, v1.y, v1.z, v1.w) << 16);
        }
        __syncthreads();

        // ---- (3) slots: one per part ----------------------------------------------------------------------------------
        bool active = lt && tid < r;
        const int ls = active ? o0 - base : 0;
        int le = active ? o1 - base : 0;
        bool bad_utf8 = false;
        if (active && P.strip_eol && le > ls) {
            le = strip_terminator(tile, ls, le, P.strip_eol);
            if (P.line_invalid != nullptr && P.line_invalid[i]) bad_utf8 = true;
        }
        const bool walk = active && !bad_utf8;
        const uint32_t nb = walk ? (uint32_t)lt_count_tabs(bmT, ls, le) + 1u : 0u;
        uint32_t slots_total;
        const uint32_t slot0 = block_exclusive_scan(nb, scan_ws, slots_total);
        if (slots_total > (uint32_t)kStageSlots) {  // CTA-uniform, rare: keep the lines whose slots fit, redo the rest next round
            const int r2 = __syncthreads_count(active && slot0 + nb <= (uint32_t)kStageSlots);
            if (r2 == 0) {  // the first line alone has more parts than there are slots: direct path
                direct_next = true;
                __syncthreads();
                continue;
            }
            r = r2;
            active = lt && tid < r;
        }
        const bool mine = walk && active;
        if (lt) {
            L.ls[tid] = ls;
            L.slot0[tid] = slot0;
            L.nb[tid] = mine ? nb : 0u;
            L.host_s[tid] = L.msg_s[tid] = L.time_s[tid] = L.level_s[tid] = 0u;
            L.dups[tid] = 0u;
            L.flags[tid] = 0u;
            L.err[tid] = 0xFFFFFFFFu;
            L.dense0[tid] = 0u;
            L.t_a[tid] = -1;
            L.t_b[tid] = 0;
            L.ts_ok[tid] = 0u;
            if (tid < 4) L.tcount[tid] = 0u;
            if (tid < 5) L.ycount[tid] = L.ypos[tid] = 0u;
            L.state[tid] = active ? 0u : 2u;
            if (tid == r - 1) s_slots = slot0 + (mine ? nb : 0u);
            if (tid == 0) s_direct = 0u;
        }
        if (mine) {
            lt_list_tabs(bmT, ls, le, tabs + slot0);
            for (uint32_t k = 0; k < nb; ++k) slot_line[slot0 + k] = (uint8_t)tid;
        }
        __syncthreads();
        const uint32_t nslots = s_slots;

        // ---- (4) one thread per part ----------------------------------------------------------------------------------
        for (uint32_t sb = 0; sb < nslots; sb += (uint32_t)kThreads) {  // warp w takes the 32 slots [sb + 32 w, sb + 32 w + 32)
            const uint32_t s = sb + (uint32_t)tid;
            bool is_row = false;
            if (s < nslots) {
                const uint32_t l = slot_line[s];
                const uint32_t k = s - L.slot0[l];
                const int start = k == 0u ? L.ls[l] : (int)tabs[s - 1] + 1;
                const int end = (int)tabs[s];
                const LtPart pt = lt_part<TYPED>(tile, start, end, cfg, S);
                stage[s] = pt.row;
                is_row = pt.kind == LP_ROW;
                if (TYPED && ((pt.row >> 56) & 0x07u) != 0u) atomicAdd(&L.ycount[(pt.row >> 56) & 0x07u], 1u);
                if (!is_row) {  // ~4 of 20 parts
                    if (pt.kind == LP_NONE) atomicOr(&L.flags[l], 0x02u);  // FG_FLAG_MISSING_VALUE: println! at :99 is replayed by the host
                    else if (pt.kind == LP_HOST) atomicMax(&L.host_s[l], s + 1u);
                    else if (pt.kind == LP_MSG) atomicMax(&L.msg_s[l], s + 1u);
                    else if (pt.kind == LP_TIME) { atomicMax(&L.time_s[l], s + 1u); atomicAdd(&L.dups[l], 1u); }
                    else { atomicMax(&L.level_s[l], s + 1u); atomicAdd(&L.dups[l], 0x100u); }
                }
            }
            const uint32_t bal = __ballot_sync(0xFFFFFFFFu, is_row);
            if (lane == 0 && sb + 32u * wid < (uint32_t)kStageSlots) L.rowmask[(sb >> 5) + wid] = bal;
        }
        __syncthreads();

        // ---- (5) values.  a: one thread per typed row; one thread per line lists its `time` value by kind ------------------
        if (TYPED) {
            // typed values differ wildly in cost (bool: a compare, f64: Rust's from_str): the typed rows are grouped by
            // type (counting sort over the slots), so that the lanes of a warp run the SAME value parser
            if (tid == 0) {
                uint32_t acc = 0;
                for (int t = 1; t < 5; ++t) { L.ybase[t] = acc; acc += L.ycount[t]; }
                L.ybase[0] = acc;  // total
            }
            __syncthreads();
            for (uint32_t s = (uint32_t)tid; s < nslots; s += (uint32_t)kThreads) {
                const uint32_t type = (uint32_t)(stage[s] >> 56) & 0x07u;
                if (type != 0u) ylist[L.ybase[type] + atomicAdd(&L.ypos[type], 1u)] = (uint16_t)s;
            }
            __syncthreads();
            const uint32_t ntyped = L.ybase[0];
            for (uint32_t q = (uint32_t)tid; q < ntyped; q += (uint32_t)kThreads) {
                const uint32_t s = ylist[q];
                const unsigned long long e = stage[s];
                const int type = (int)((e >> 56) & 0x07u);
                const int va = (int)(e & 0xFFFFu) + (int)((e >> 16) & 0xFFFFu) + 1;
                unsigned long long val = 0;
                const uint32_t st = ltsv_parse_typed(tile, va, va + (int)((e >> 32) & 0xFFFFFFu), type, val);
                if (st == FG_ST_OK) stage_val[s] = val;
                else {
                    const uint32_t l = slot_line[s];
                    atomicMin(&L.err[l], ((s - L.slot0[l]) << 8) | st);
                }
            }
        }
        // value bounds of a special part: slot s covers [start, tabs[s]), the value starts behind `key:`
        auto value_of = [&](uint32_t s1, int key_len, int& a, int& b, int& k) {
            a = -1; b = 0; k = -1;
            if (s1 == 0u) return;
            const uint32_t s = s1 - 1u;
            k = (int)(s - slot0);
            const int start = k == 0 ? ls : (int)tabs[s - 1] + 1;
            a = start + key_len + 1;
            b = (int)tabs[s];
        };
        bool direct = false;
        int t_a = -1, t_b = 0, t_k = -1;
        if (mine) {
            const uint32_t d = L.dups[tid];
            // a repeated `time` / `level`: every occurrence is evaluated in order (:104-121) — round-1 scanner
            direct = (d & 0xFFu) > 1u || (d >> 8) > 1u;
            if (!direct) {
                value_of(L.time_s[tid], 4, t_a, t_b, t_k);
                if (t_a >= 0) {
                    L.t_a[tid] = t_a;
                    L.t_b[tid] = t_b;
                    const int c = lt_time_class(tile, t_a, t_b);
                    L.tlist[c][atomicAdd(&L.tcount[c], 1u)] = (uint32_t)tid;
                }
            }
        }
        __syncthreads();
        // b: parse_ts — warps 2c and 2c + 1 take the lines of class c, so the four attempts of :263-267 run side by side on
        // different warps instead of one after the other on the same lanes
        {
            const uint32_t idx = ((wid & 1u) << 5) + lane;
            for (uint32_t c = wid >> 1; c < 4u; c += (uint32_t)kWarps >> 1) {  // 8 warps: one pair per class
                if (idx < L.tcount[c]) {
                    const uint32_t l = L.tlist[c][idx];
                    double ts;
                    const bool ok = lt_time_value(tile, L.t_a[l], L.t_b[l], ts);
                    L.ts[l] = ts;
                    L.ts_ok[l] = ok ? 1u : 0u;
                }
            }
        }
        __syncthreads();
        // c: one thread per line settles the status
        LineResult res;
        res.ts = 0.0;
        res.facility = 0xFFu;
        res.severity = 0xFFu;
        res.flags = 0;
        res.status = FG_ST_OK;
        res.host_o = res.app_o = res.proc_o = res.mid_o = res.msg_o = res.full_o = -1;
        res.host_l = res.app_l = res.proc_l = res.mid_l = res.msg_l = res.full_l = 0;
        res.n_entries = 0;
        uint32_t my_n = 0;
        if (mine) {
            if (!direct) {
                int l_a, l_b, l_k, h_a, h_b, h_k, m_a, m_b, m_k;
                value_of(L.level_s[tid], 5, l_a, l_b, l_k);
                value_of(L.host_s[tid], 4, h_a, h_b, h_k);
                value_of(L.msg_s[tid], 7, m_a, m_b, m_k);
                const int bad_k = lt_finish_line(tile, t_k, L.ts_ok[tid] != 0u, L.ts[tid], l_a, l_b, l_k, L.err[tid], h_a >= 0, res);
                res.flags = L.flags[tid];
                if (res.status == FG_ST_OK) {
                    if (h_a >= 0) { res.host_o = h_a - ls; res.host_l = h_b - h_a; }
                    if (m_a >= 0) { res.msg_o = m_a - ls; res.msg_l = m_b - m_a; }
                    res.full_o = 0;  // full_msg = the whole line, untrimmed :219
                    res.full_l = le - ls;
                    my_n = lt_rows_between(L.rowmask, slot0, slot0 + nb);
                } else {
                    // the failing part (LTSV side effects on the host stop there); a missing timestamp / hostname: after the last part
                    res.full_o = bad_k >= 0 ? (bad_k == 0 ? ls : (int)tabs[slot0 + (uint32_t)bad_k - 1u] + 1) - ls : (le - ls) + 1;
                    res.severity = 0xFFu;
                    res.ts = 0.0;
                }
            }
            L.state[tid] = direct ? 1u : (res.status == FG_ST_OK ? 0u : 3u);
            if (direct) atomicAdd(&s_direct, 1u);
        }
        if (bad_utf8) {
            res.status = FG_ES_INVALID_UTF8;
            res.full_o = 0;
            if (active) L.state[tid] = 3u;
        }

        // ---- (6) rows of the decoded lines: place (scan over the lines + ONE global atomic), write --------------------------
        uint32_t total;
        const uint32_t excl = block_exclusive_scan(my_n, scan_ws, total);  // (its barriers also publish L.state)
        if (lt) L.dense0[tid] = excl;
        if (tid == 0 && total) s_ebase = atomicAdd(P.entry_counter, total);
        __syncthreads();
        const uint32_t ebase = total ? s_ebase : 0u;
        const bool ovf = (unsigned long long)ebase + total > (unsigned long long)P.entry_cap;
        if (total && !ovf) {
            // one thread per slot; a row's place = rows of its line before it (popcount over the row mask)
            for (uint32_t s = (uint32_t)tid; s < nslots; s += (uint32_t)kThreads) {
                const unsigned long long e = stage[s];
                if (e == 0ull) continue;
                const uint32_t l = slot_line[s];
                if (L.state[l] != 0u) continue;
                const uint32_t j = ebase + L.dense0[l] + lt_rows_between(L.rowmask, L.slot0[l], s);
                const int ka = base + (int)(e & 0xFFFFu), kn = (int)((e >> 16) & 0xFFFFu);
                const uint32_t meta = (uint32_t)(e >> 56) & 0x7Fu;  // without kLtRow
                sink.name[j] = make_int2(ka, kn);
                unsigned long long v = (unsigned long long)(uint32_t)(ka + kn + 1) | (((e >> 32) & 0xFFFFFFull) << 32);
                if (TYPED && (meta & 0x07u) != 0u) v = stage_val[s];
                sink.val[j] = v;
                sink.meta[j] = (uint8_t)meta;
            }
        }
        if (active && !direct) {
            const uint32_t n_out = ovf ? 0u : my_n;
            write_row(P, i, o0, res, n_out ? ebase + excl : 0u, n_out);
        }

        // ---- lines of this round that need the sequential scanner (CTA-uniform loop, rare) -----------------------------
        if (s_direct) {
            for (int l = 0; l < r; ++l)
                if (L.state[l] == 1u) direct_line(P, cur + l, sink, tmp);  // shared memory: the same for every thread
        }
        __syncthreads();  // tile, bitmap, slots and the line records are reused by the next round
        cur += r;
    }
}

}  // namespace

int parse_ltsv_smem_bytes(int tile_bytes, bool typed) {
    return tile_bytes + (tile_bytes / 32 + 4) * 4 + kLtsvStageSlots * 8 * (typed ? 2 : 1) + kLtsvStageSlots * 2 * (typed ? 2 : 1) + kLtsvStageSlots + 16;
}

cudaError_t configure_parse_ltsv(int max_tile_bytes) {
    cudaError_t e = cudaFuncSetAttribute(parse_ltsv_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         parse_ltsv_smem_bytes(max_tile_bytes, false));
    if (e != cudaSuccess) return e;
    return cudaFuncSetAttribute(parse_ltsv_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                parse_ltsv_smem_bytes(max_tile_bytes, true));
}

cudaError_t launch_parse_ltsv(const ParseParams& p, cudaStream_t stream) {
    if (p.n <= 0) return cudaSuccess;
    if (p.tile_bytes <= 0 || p.tile_bytes > kLtsvMaxTile || (p.tile_bytes & 511)) return cudaErrorInvalidValue;
    const int grid = (p.n + kLines - 1) / kLines;
    const bool typed = p.ltsv.has_schema != 0;
    if (typed) parse_ltsv_kernel<true><<<grid, kThreads, parse_ltsv_smem_bytes(p.tile_bytes, true), stream>>>(p);
    else parse_ltsv_kernel<false><<<grid, kThreads, parse_ltsv_smem_bytes(p.tile_bytes, false), stream>>>(p);
    return cudaGetLastError();
}

}  // namespace fg
