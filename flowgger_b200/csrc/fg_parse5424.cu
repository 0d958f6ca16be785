// fg_parse5424.cu — the RFC5424 hot path on sm_90a: bytes -> compact 32-byte rows + 8-byte side-table entries.
//
//   parse5424_kernel     one CTA = LINES consecutive lines.  (1) thread 0 issues ONE TMA bulk copy (cp.async.bulk, SASS
//                        UBLKCP) of the CTA's contiguous byte span into the shared-memory tile; (2) all threads sweep the tile
//                        16 bytes per step and write the structural bitmap (fg_r5fast.cuh stage 1: coalesced, conflict-free,
//                        32 of 32 lanes busy); (3) one thread per line walks its line hop by hop over the bitmap (stage 2,
//                        lock step) and stages its side-table rows inside its own consumed bytes; (4) a CTA scan + ONE global
//                        atomic place the rows, which are copied out with the 32-byte row of every line.
//   post5424_kernel      one launch for the two device-side work lists:
//     unescape_lines     the few lines (≈8 % at C2) whose SD values hold a backslash: unescape_sd_value
//                        (rfc5424_decoder.rs:105-125) into the batch arena, one thread per listed line;
//     wide_lines         the SLOW path: every line the fast walker does not recognise as regular (malformed lines and
//                        their error strings, legal-but-unusual shapes, lines >= 64 KiB or longer than the tile, rows that
//                        do not fit behind the cursor) goes through the exact scanner of fg_rfc5424.cuh straight from
//                        global memory (≈0.6 % of the lines at C2).
// The work lists live on the device, so a batch needs no host round trip between the two launches.
#include "fg_kernels.cuh"

#include "fg_common.cuh"
#include "fg_r5fast.cuh"
#include "fg_rfc5424.cuh"
#include "fg_status.h"
#include "fg_tma.cuh"

namespace fg {

namespace {

constexpr int kFastLines = kRfc5424LinesPerCta;  // lines (= threads) per CTA
constexpr int kFastCtasPerSm = kRfc5424CtasPerSm;

template <int LINES, int MINB>
__global__ void __launch_bounds__(LINES, MINB) parse5424_kernel(const __grid_constant__ Parse5424Params P) {
    extern __shared__ __align__(128) uint8_t tile[];
    __shared__ __align__(8) uint64_t mbar;
    __shared__ uint32_t scan_ws[2 * (LINES / 32)];  // per-warp totals of the two packed counters
    __shared__ uint32_t s_base[3];                  // side-table base, escape-list base, wide-list base of this round

    const int tid = threadIdx.x;
    const uint32_t lane = (uint32_t)tid & 31u;
    const int first = blockIdx.x * LINES;
    const int last = min(P.n, first + LINES);
    // the bitmap I ("may end a token") lives behind the tile: tile_bytes / 8 + 16 bytes
    uint32_t* bmI = reinterpret_cast<uint32_t*>(tile + P.tile_bytes);
    if (*P.bad_offsets) return;  // CTA-uniform
    if (tid == 0) mbar_init(&mbar, 1);
    __syncthreads();

    uint32_t parity = 0;
    int cur = first;
    while (cur < last) {
        const int i = cur + tid;
        const int o0 = __ldg(P.offsets + min(i, last));
        const int o1 = __ldg(P.offsets + min(i + 1, last));
        const int ocur = __ldg(P.offsets + cur);
        const int base = ocur & ~15;
        const bool fits = (i < last) && (o1 - base <= P.tile_bytes);
        const int r = __syncthreads_count(fits);  // offsets are monotone: `fits` is a prefix property
        if (r == 0) {
            // the first pending line alone exceeds the tile: the wide kernel takes it
            if (tid == 0) P.wide_list[atomicAdd(P.counters + K5_WIDE_LIST, 1u)] = (uint32_t)cur;
            cur += 1;
            continue;
        }
        const int oend = __ldg(P.offsets + cur + r);
        const uint32_t nbytes = (uint32_t)((oend - base) + 15) & ~15u;
        if (tid == 0) {
            fence_proxy_async();  // generic-proxy accesses of the previous round happen-before this async write
            mbar_expect_tx(&mbar, nbytes);
            bulk_g2s(tile, P.bytes + base, nbytes, &mbar);
        }
        mbar_wait(&mbar, parity);
        parity ^= 1u;

        // ---- stage 1: structural bitmap of the whole tile, 32 bytes (= one bitmap word) per thread per step -------
        const int nword = (int)((nbytes + 31u) >> 5);  // the tile allocation is a multiple of 512 bytes: reading the odd granule is safe
        for (int g = tid; g < nword; g += LINES) {
            const uint4 v0 = reinterpret_cast<const uint4*>(tile)[2 * g], v1 = reinterpret_cast<const uint4*>(tile)[2 * g + 1];
            bmI[g] = r5_classify16(v0.x, v0.y, v0.z, v0.w) | (r5_classify16(v1.x, v1.y, v1.z, v1.w) << 16);
        }
        if (tid < 3) bmI[nword + tid] = 0;  // r5_window reads up to two words past the last one
        __syncthreads();

        // ---- stage 2: one thread per line ------------------------------------------------------------------------
        // (Counting-sorting the CTA's lines by a work estimate so that a warp's 32 lines have similar pair counts was
        //  slower: the estimate, the two extra barriers and the scattered row stores cost more than the shorter walks gain.)
        const bool active = tid < r;
        int ls = active ? o0 - base : 0;
        int le = active ? o1 - base : 0;
        bool bad_utf8 = false;
        if (P.strip_eol && le > ls) {
            // BufRead::lines: drop the '\n' and one '\r' before it (line_splitter.rs:17); invalid UTF-8 lines are skipped (:22-25)
            if (P.strip_eol == 2) {  // BufRead::split(0): only the NUL terminator goes (nul_splitter.rs:18)
                if (tile[le - 1] == 0) --le;
            } else if (tile[le - 1] == '\n') {
                --le;
                if (le > ls && tile[le - 1] == '\r') --le;
            }
            if (P.line_invalid != nullptr && P.line_invalid[i]) bad_utf8 = true;
        }
        const bool too_long = le - ls > 65535;
        R5Fast res;
        const bool regular = r5_regular(tile, bmI, ls, (too_long || bad_utf8 || !active) ? ls : le, res);
        if (bad_utf8) {
            res.status = FG_ES_INVALID_UTF8;
            res.n_entries = 0;
        }
        // anything that is not a regular line (malformed, unusual but legal, 64 KiB or longer) is redone by the slow kernel
        const bool wide = active && !regular && !bad_utf8;
        const uint32_t my_n = (active && !wide && res.status == FG_ST_OK) ? res.n_entries : 0u;
        const bool esc = my_n != 0u && res.esc;

        // Placement of this round's output: ONE scan over two packed counters per line — side-table rows, and
        // (escape-list | wide-list << 8) memberships — then one global atomic per non-empty counter, issued by three
        // different threads so that their round trips overlap.
        uint32_t xa = my_n, xb = (esc ? 1u : 0u) | (wide ? 0x100u : 0u);
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
            const uint32_t ya = __shfl_up_sync(0xFFFFFFFFu, xa, d), yb = __shfl_up_sync(0xFFFFFFFFu, xb, d);
            if (lane >= (uint32_t)d) { xa += ya; xb += yb; }
        }
        const int wid = tid >> 5;
        constexpr int kWarps = LINES / 32;
        if (lane == 31u) { scan_ws[wid] = xa; scan_ws[kWarps + wid] = xb; }
        __syncthreads();
        uint32_t before_a = 0, before_b = 0, total = 0, total_b = 0;
#pragma unroll
        for (int w = 0; w < kWarps; ++w) {
            const uint32_t ta = scan_ws[w], tb = scan_ws[kWarps + w];
            if (w < wid) { before_a += ta; before_b += tb; }
            total += ta;
            total_b += tb;
        }
        const uint32_t excl = before_a + xa - my_n;
        const uint32_t pos_b = before_b + xb - ((esc ? 1u : 0u) | (wide ? 0x100u : 0u));  // exclusive: esc rank | wide rank << 8
        const uint32_t n_esc = total_b & 0xFFu, n_wide = total_b >> 8;
        if (total | total_b) {  // CTA-uniform
            if (tid == 0 && total) s_base[0] = atomicAdd(P.counters + K5_ENTRIES, total);
            if (tid == 32 % LINES && n_esc) s_base[1] = atomicAdd(P.counters + K5_ESC_LIST, n_esc);
            if (tid == 33 % LINES && n_wide) s_base[2] = atomicAdd(P.counters + K5_WIDE_LIST, n_wide);
            __syncthreads();
        }
        const uint32_t esc_at = pos_b & 0xFFu, wide_at = pos_b >> 8;
        uint32_t my_begin = 0;
        if (my_n) {
            my_begin = s_base[0] + excl;
            if ((unsigned long long)my_begin + my_n <= (unsigned long long)P.entry_cap) {
                unsigned long long* dst = P.entries + my_begin;
                for (uint32_t k = 0; k < my_n; ++k) dst[k] = res.stage[k];
            }
        }
        if (esc) P.esc_list[s_base[1] + esc_at] = (uint32_t)i;
        if (wide) P.wide_list[s_base[2] + wide_at] = (uint32_t)i;
        if (active && !wide) {
            const bool ok = res.status == FG_ST_OK;
            const uint32_t meta = ok ? (res.facility << 8) | (res.severity << 16) | (res.flags << 24) : res.status | 0x00FFFF00u;
            uint4 lo4, hi4;
            lo4.x = (uint32_t)__double2loint(res.ts);
            lo4.y = (uint32_t)__double2hiint(res.ts);
            lo4.z = meta;
            lo4.w = my_begin;
            hi4.x = my_n | ((uint32_t)res.sp1 << 16);
            hi4.y = (uint32_t)res.sp2 | ((uint32_t)res.sp3 << 16);
            hi4.z = (uint32_t)res.sp4 | ((uint32_t)res.sp5 << 16);
            hi4.w = (uint32_t)res.msg_o | ((uint32_t)res.msg_l << 16);
            if (!ok) {
                lo4.x = lo4.y = 0u;
                hi4 = make_uint4(0u, 0u, 0u, 0u);
            }
            P.rows[2 * (size_t)i] = lo4;
            P.rows[2 * (size_t)i + 1] = hi4;
        }
        __syncthreads();  // tile, bitmap and scan scratch are reused by the next round
        cur += r;
    }
}

// One thread per listed line, ONE pass: the arena bytes are reserved from the raw lengths (an unescaped value is never
// longer than the raw one; a record is [u16 length][bytes], 2-byte aligned) with one warp-aggregated atomic, then every
// escaped value is rewritten and its side-table row switched to the arena form.
__device__ __forceinline__ void unescape_lines(const Parse5424Params& P, uint32_t first_item, uint32_t stride) {
    const uint32_t cnt = P.counters[K5_ESC_LIST];
    const uint32_t lane = threadIdx.x & 31u;
    for (uint32_t j0 = first_item; j0 < cnt; j0 += stride) {
        const uint32_t j = j0 + lane;
        const bool valid = j < cnt;
        uint32_t first = 0, count = 0;
        int o0 = 0;
        if (valid) {
            const uint32_t line = P.esc_list[j];
            const uint4 lo4 = P.rows[2 * (size_t)line], hi4 = P.rows[2 * (size_t)line + 1];
            o0 = P.offsets[line];
            first = lo4.w;
            count = hi4.x & 0xFFFFu;
            if ((unsigned long long)first + count > (unsigned long long)P.entry_cap) count = 0;  // side table overflowed: the batch is redone
        }
        uint32_t need = 0;
        for (uint32_t e = 0; e < count; ++e) {
            const unsigned long long v = P.entries[first + e];
            if (!(v & kE8Header) && (v & kE8Esc)) need += (2u + (uint32_t)((v >> 32) & 0xFFFFu) - ((uint32_t)((v >> 16) & 0xFFFFu) + 2u) + 1u) & ~1u;
        }
        uint32_t inc = need;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
            const uint32_t y = __shfl_up_sync(0xFFFFFFFFu, inc, d);
            if (lane >= (uint32_t)d) inc += y;
        }
        const uint32_t warp_total = __shfl_sync(0xFFFFFFFFu, inc, 31);
        uint32_t abase = 0;
        if (lane == 0 && warp_total) abase = atomicAdd(P.counters + K5_ARENA, warp_total);
        abase = __shfl_sync(0xFFFFFFFFu, abase, 0);
        if ((unsigned long long)abase + warp_total > (unsigned long long)P.arena_cap) continue;  // arena overflowed: the batch is redone
        // The values are rewritten in lock step: round j handles every lane's j-th escaped value, and inside a round the
        // 32 lanes consume one raw byte per iteration together (a lane per value with its own byte loop ran ~3 lanes wide).
        uint32_t at = abase + inc - need;
        uint32_t e = 0;
        for (;;) {
            // next escaped pair of this lane
            unsigned long long v = 0;
            bool have = false;
            for (; e < count; ++e) {
                v = P.entries[first + e];
                if (!(v & kE8Header) && (v & kE8Esc)) { have = true; break; }
            }
            if (!__any_sync(0xFFFFFFFFu, have)) break;
            const int ne = (int)((v >> 16) & 0xFFFFu), ve = (int)((v >> 32) & 0xFFFFu);
            const int len = have ? ve - (ne + 2) : 0;
            const uint8_t* src = P.bytes + o0 + ne + 2;
            uint8_t* dst = P.arena + at + 2;
            int k = 0, o = 0;
            while (__any_sync(0xFFFFFFFFu, k < len)) {
                if (k < len) {
                    const uint32_t c = src[k++];
                    if (c != '\\') {
                        dst[o++] = (uint8_t)c;
                    } else if (k < len) {  // a trailing lone backslash is dropped (rfc5424_decoder.rs:105-125)
                        const uint32_t d = src[k++];
                        if (d != '"' && d != '\\' && d != ']') dst[o++] = '\\';
                        dst[o++] = (uint8_t)d;
                    }
                }
            }
            if (have) {
                *reinterpret_cast<uint16_t*>(P.arena + at) = (uint16_t)o;
                P.entries[first + e] = (v & 0xFFFFFFFFull) | ((unsigned long long)(at >> 1) << 32) | kE8Arena;
                at += (2u + (uint32_t)len + 1u) & ~1u;
                ++e;
            }
        }
    }
}

// The round-1 scanner over the listed lines, one thread per line straight from global memory: a counting pass, one
// atomic per line for its side-table rows, an emitting pass, then the unescape of its values and the wide row.
__device__ __forceinline__ void wide_lines(const Parse5424Params& P, int (*marks)[32], uint32_t first_item, uint32_t stride) {
    const uint32_t cnt = P.counters[K5_WIDE_LIST];
    const uint32_t lane = threadIdx.x & 31u;
    const EntrySink sink = {P.wentry_name, P.wentry_val, P.wentry_meta};
    for (uint32_t j0 = first_item; j0 < cnt; j0 += stride) {
        const uint32_t j = j0 + lane;
        const bool valid = j < cnt;
        uint32_t line = 0;
        int o0 = 0, len = 0;
        bool bad_utf8 = false;
        if (valid) {
            line = P.wide_list[j];
            o0 = P.offsets[line];
            len = P.offsets[line + 1] - o0;
            if (P.strip_eol && len > 0) {
                if (P.strip_eol == 2) {
                    if (P.bytes[o0 + len - 1] == 0) --len;
                } else if (P.bytes[o0 + len - 1] == '\n') {
                    --len;
                    if (len > 0 && P.bytes[o0 + len - 1] == '\r') --len;
                }
                if (P.line_invalid != nullptr && P.line_invalid[line]) bad_utf8 = true;
            }
            if (bad_utf8) len = 0;
        }
        LineResult res;
        rfc5424_parse_line<32>(P.bytes + o0, len, o0, &marks[0][lane], res, sink, 0u, false);
        uint32_t n = (valid && !bad_utf8 && res.status == FG_ST_OK) ? res.n_entries : 0u;
        uint32_t wbase = 0;
        if (n) {
            wbase = atomicAdd(P.counters + K5_WIDE_ENTRIES, n);
            if ((unsigned long long)wbase + n > (unsigned long long)P.wentry_cap) n = 0;  // table overflowed: the batch is redone
        }
        {
            LineResult again;  // same fields as `res`; only the rows matter (lanes without rows run an empty line)
            rfc5424_parse_line<32>(P.bytes + o0, n ? len : 0, o0, &marks[0][lane], again, sink, wbase, true);
        }
        if (!valid) continue;
        // unescape_sd_value (:105-125) of the flagged values into the arena
        for (uint32_t k = 0; k < n; ++k) {
            const uint32_t e = wbase + k;
            const uint8_t m = sink.meta[e];
            if ((m & 0x07u) == 0u && (m & 0x08u)) {
                const unsigned long long v = sink.val[e];
                const uint32_t off = (uint32_t)v, l = (uint32_t)(v >> 32);
                const uint32_t ul = (uint32_t)r5_unescape(P.bytes + off, (int)l, nullptr);
                const uint32_t at = atomicAdd(P.counters + K5_ARENA, (ul + 1u) & ~1u);  // keeps the arena 2-byte aligned for the [u16 length] records
                if ((unsigned long long)at + ul <= (unsigned long long)P.arena_cap) r5_unescape(P.bytes + off, (int)l, P.arena + at);
                sink.val[e] = (unsigned long long)at | ((unsigned long long)ul << 32);
                sink.meta[e] = (uint8_t)0x80u;  // FG_TAG_STRING | FG_EM_ARENA
            }
        }
        if (bad_utf8) {
            res.status = FG_ES_INVALID_UTF8;
            res.flags = 0;
            res.facility = res.severity = 0xFFu;
        }
        const bool ok = res.status == FG_ST_OK;
        if (!ok) {  // an error row is its status, nothing else
            P.rows[2 * (size_t)line] = make_uint4(0u, 0u, res.status | 0x00FFFF00u, 0u);
            P.rows[2 * (size_t)line + 1] = make_uint4(0u, 0u, 0u, 0u);
            continue;
        }
        const uint32_t widx = atomicAdd(P.counters + K5_WIDE_ROWS, 1u);
        const uint32_t meta = res.status | (res.facility << 8) | (res.severity << 16) | ((res.flags | kFlagWide) << 24);
        if (widx < P.wide_cap) {
            WideRow w;
            w.line = P.line0 + (int32_t)line;
            w.meta = meta;
            w.ts = res.ts;
            w.host = make_int2(ok ? o0 + res.host_o : -1, res.host_l);
            w.app = make_int2(ok ? o0 + res.app_o : -1, res.app_l);
            w.proc = make_int2(ok ? o0 + res.proc_o : -1, res.proc_l);
            w.msgid = make_int2(ok ? o0 + res.mid_o : -1, res.mid_l);
            w.msg = make_int2(ok && res.msg_o >= 0 ? o0 + res.msg_o : -1, res.msg_l);
            w.full = make_int2(ok && res.full_o >= 0 ? o0 + res.full_o : -1, res.full_l);
            w.sd = make_int2((int)wbase, (int)(ok ? n : 0u));
            P.wide_rows[widx] = w;
        }
        P.rows[2 * (size_t)line] = make_uint4((uint32_t)__double2loint(res.ts), (uint32_t)__double2hiint(res.ts), meta, widx);
        P.rows[2 * (size_t)line + 1] = make_uint4(0u, 0u, 0u, 0u);
    }
}

// ONE launch after the parse kernel for both device-side work lists: the first `esc_ctas` CTAs rewrite the escaped values
// (unescape_lines), the remaining CTAs run the slow exact scanner over the irregular lines (wide_lines) — the two lists
// are independent, so they share the machine instead of queueing behind each other.
__global__ void __launch_bounds__(128) post5424_kernel(const __grid_constant__ Parse5424Params P, int esc_ctas) {
    __shared__ int marks[4][6][32];
    if (*P.bad_offsets) return;
    const uint32_t warp = threadIdx.x >> 5;
    if ((int)blockIdx.x < esc_ctas) {
        unescape_lines(P, (blockIdx.x * 4u + warp) * 32u, (uint32_t)esc_ctas * 128u);
    } else {
        const uint32_t wctas = gridDim.x - (uint32_t)esc_ctas;
        wide_lines(P, marks[warp], ((blockIdx.x - (uint32_t)esc_ctas) * 4u + warp) * 32u, wctas * 128u);
    }
}

}  // namespace

int parse5424_smem_bytes(int tile_bytes) { return tile_bytes + tile_bytes / 8 + 16; }

cudaError_t configure_parse5424(int max_tile_bytes) {
    return cudaFuncSetAttribute(parse5424_kernel<kFastLines, kFastCtasPerSm>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                parse5424_smem_bytes(max_tile_bytes));
}

cudaError_t launch_parse5424(const Parse5424Params& p, cudaStream_t stream, cudaEvent_t dom0, cudaEvent_t dom1) {
    if (p.n <= 0) return cudaSuccess;
    const int grid = (p.n + kFastLines - 1) / kFastLines;
    if (dom0) cudaEventRecord(dom0, stream);
    parse5424_kernel<kFastLines, kFastCtasPerSm><<<grid, kFastLines, parse5424_smem_bytes(p.tile_bytes), stream>>>(p);
    if (dom1) cudaEventRecord(dom1, stream);
    // the work lists live on the device (no host round trip): a fixed grid strides over them
    const long long sms = p.num_sms;
    const int esc_ctas = (int)min((long long)(p.n + 127) / 128, sms * 12);
    const int wide_ctas = (int)min((long long)(p.n + 127) / 128, sms * 4);
    post5424_kernel<<<esc_ctas + wide_ctas, 128, 0, stream>>>(p, esc_ctas);
    return cudaGetLastError();
}

}  // namespace fg
