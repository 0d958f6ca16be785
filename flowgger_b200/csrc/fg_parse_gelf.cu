// fg_parse_gelf.cu — the GELF decoder on sm_90a: bytes -> row columns + side table, on the bitmap pipeline, member-parallel.
//
//   parse_gelf_kernel   one CTA = 64 consecutive lines, 256 threads.  Per round:
//     (1) ONE TMA bulk copy (cp.async.bulk, SASS UBLKCP) of the lines' contiguous byte span into the shared-memory tile;
//     (2) all threads sweep the tile 32 bytes per step into three bitmaps — quotes, backslashes, commas — and a
//         control-byte flag per granule (fg_gelffast.cuh stage 1);
//     (3) one thread per line runs over the line's bitmap WORDS: escaped quotes, string interior, the commas outside
//         strings = member boundaries; a CTA scan gives every member a SLOT;
//     (4) one thread per SLOT (all 256 threads) validates and converts its member: key, colon, string escapes, literals;
//         number tokens are listed and parsed by a dense second pass (json_number on 32 busy lanes);
//     (5) one thread per line: BTreeMap order, last duplicate wins, the per-key rules (gelf_decoder.rs:51-110); the rows it
//         keeps are written over the line's own slots;
//     (6) a second scan + ONE global atomic place the rows and all threads copy them out — consecutive threads write
//         consecutive rows of the three side-table columns.
//     Lines that are not regular (fg_gelffast.cuh) go on a device-side list.
//   post_gelf_kernel    the SLOW path over that list: the exact parser of fg_gelf.cuh (the whole serde_json grammar, the
//                       newline retry, every error string), one thread per listed line straight from global memory.
#include "fg_kernels.cuh"

#include "fg_common.cuh"
#include "fg_gelffast.cuh"
#include "fg_status.h"
#include "fg_tma.cuh"

#include <cstdio>
#include <cstdlib>

namespace fg {

namespace {

constexpr int kLines = kGelfLinesPerCta;
constexpr int kThreads = kGelfThreadsPerCta;
constexpr int kSlots = kGelfStageSlots;
constexpr int kCtrlWords = (kGelfMaxTile / 32 / 32 + 8 + 3) & ~3;  // one bit per 32-byte granule of the largest tile; keeps the slots 16-byte aligned

__device__ __forceinline__ void write_row(const ParseParams& P, int i, int o0, const LineResult& res, uint32_t my_begin, uint32_t my_n) {
    const bool ok = res.status == FG_ST_OK;
    P.ts[i] = res.ts;
    P.meta[i] = res.status | (res.facility << 8) | (res.severity << 16) | (res.flags << 24);
    P.host[i] = make_int2(res.host_o >= 0 ? o0 + res.host_o : -1, res.host_l);
    P.msg[i] = make_int2(res.msg_o >= 0 ? o0 + res.msg_o : -1, res.msg_l);
    P.full[i] = ok ? make_int2(res.full_o >= 0 ? o0 + res.full_o : -1, res.full_l) : make_int2(o0 + max(res.full_o, 0), 0);
    P.sd[i] = make_int2((int)my_begin, (int)my_n);
}

__global__ void __launch_bounds__(kThreads, kGelfCtasPerSm) parse_gelf_kernel(const __grid_constant__ ParseParams P) {
    extern __shared__ __align__(128) uint8_t tile[];
    __shared__ __align__(8) uint64_t mbar;
    __shared__ uint32_t scan_ws[33];
    __shared__ uint32_t s_ebase, s_slots, s_slow_base, s_nnum, s_nlong;
    __shared__ int line_ls[kLines], line_o0[kLines], line_open[kLines];
    __shared__ uint32_t line_slot[kLines];   // first slot | members (later: rows) << 16
    __shared__ uint32_t line_dense[kLines];  // exclusive sum of the rows of the lines before this one
    __shared__ uint32_t line_bad[kLines];    // a member was rejected: the line goes to the exact parser

    const int tid = threadIdx.x;
    const int first = blockIdx.x * kLines;
    const int last = min(P.n, first + kLines);
    // behind the tile: three bitmaps (tile_bytes / 32 + 4 words each), the control-byte flags (one bit per 32-byte granule)
    // and the slots — first a member each, in the end the side-table rows of the line: name column, value column, meta
    // column, member end ("cut"), slot -> line map, the list of number members
    const int bm_words = P.tile_bytes / 32 + 4;
    uint32_t* bmQ = reinterpret_cast<uint32_t*>(tile + P.tile_bytes);
    uint32_t* bmB = bmQ + bm_words;
    uint32_t* bmP = bmB + bm_words;
    uint32_t* anyK = bmP + bm_words;  // kCtrlWords
    int2* st_name = reinterpret_cast<int2*>(anyK + kCtrlWords);
    unsigned long long* st_val = reinterpret_cast<unsigned long long*>(st_name + kSlots);
    uint16_t* cuts = reinterpret_cast<uint16_t*>(st_val + kSlots);
    uint16_t* numlist = cuts + kSlots;
    uint8_t* st_meta = reinterpret_cast<uint8_t*>(numlist + kSlots);
    uint8_t* slot_line = st_meta + kSlots;
    const uint32_t lane = (uint32_t)tid & 31u, wid = (uint32_t)tid >> 5;
    if (*P.bad_offsets) return;  // CTA-uniform
    if (tid == 0) mbar_init(&mbar, 1);
    __syncthreads();

    const EntrySink sink = {P.entry_name, P.entry_val, P.entry_meta};
    const EntrySink stage = {st_name, st_val, st_meta};
    uint32_t parity = 0;
    int cur = first;
    while (cur < last) {
        const bool lt = tid < kLines;  // line threads
        const int i = cur + tid;
        int o0 = 0, o1 = 0;
        if (lt) {
            o0 = __ldg(P.offsets + min(i, last));
            o1 = __ldg(P.offsets + min(i + 1, last));
        }
        const int ocur = __ldg(P.offsets + cur);
        const int base = ocur & ~15;
        const bool fits = lt && (i < last) && (o1 - base <= P.tile_bytes);
        int r = __syncthreads_count(fits);  // offsets are monotone: `fits` is a prefix property
        if (r == 0) {
            // the first pending line alone exceeds the tile: the slow kernel takes it
            if (tid == 0) P.slow_list[atomicAdd(P.slow_count, 1u)] = (uint32_t)cur;
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

        // ---- (2) the three bitmaps of the whole tile, 32 bytes (= one word of each) per thread per step ----------------------
        const int nword = (int)((nbytes + 31u) >> 5);
        for (int gb = 0; gb < nword; gb += kThreads) {  // warp w takes the 32 granules [gb + 32 w, gb + 32 w + 32)
            const int g = gb + tid;
            uint32_t ctrl = 0;
            if (g < nword) {
                const uint4 v0 = reinterpret_cast<const uint4*>(tile)[2 * g], v1 = reinterpret_cast<const uint4*>(tile)[2 * g + 1];
                uint32_t q0, b0, p0, c0, q1, b1, p1, c1;
                gf_bits16(v0.x, v0.y, v0.z, v0.w, q0, b0, p0, c0);
                gf_bits16(v1.x, v1.y, v1.z, v1.w, q1, b1, p1, c1);
                if ((uint32_t)(32 * g + 16) >= nbytes) q1 = b1 = p1 = c1 = 0u;  // the odd granule: bytes of an earlier round
                bmQ[g] = q0 | (q1 << 16);
                bmB[g] = b0 | (b1 << 16);
                bmP[g] = p0 | (p1 << 16);
                ctrl = c0 | c1;
            }
            const uint32_t bal = __ballot_sync(0xFFFFFFFFu, ctrl != 0u);
            if (lane == 0) anyK[(gb >> 5) + (int)wid] = bal;
        }
        if (tid < 4) bmQ[nword + tid] = bmB[nword + tid] = bmP[nword + tid] = 0;
        if (tid == 0) s_nnum = s_nlong = 0u;
        __syncthreads();

        // ---- (3) one thread per line: the member boundaries, from the bitmap words -----------------------------------------
        bool active = lt && tid < r;
        const int ls = active ? o0 - base : 0;
        int le = active ? o1 - base : 0;
        bool bad_utf8 = false;
        if (active && P.strip_eol && le > ls) {
            // BufRead::lines: drop the '\n' and one '\r' before it (line_splitter.rs:17); invalid UTF-8 lines are skipped (:22-25)
            if (P.strip_eol == 2) {  // BufRead::split(0): only the NUL terminator goes (nul_splitter.rs:18)
                if (tile[le - 1] == 0) --le;
            } else if (tile[le - 1] == '\n') {
                --le;
                if (le > ls && tile[le - 1] == '\r') --le;
            }
            if (P.line_invalid != nullptr && P.line_invalid[i]) bad_utf8 = true;
        }
        const bool walk = active && !bad_utf8;
        bool regular = false;
        uint32_t nm = 0;
        int open = 0;
        uint16_t my_cuts[kMaxLocalMembers];
        if (tid < kLines) {  // warp-uniform: the warps that hold line threads run the line pass in lock step
            // (a raw control byte anywhere in the line sends it to the exact parser: newline retry / error)
            const bool cand = walk && !gf_has_ctrl(tile, anyK, ls, le);
            const int m = gf_line_members(tile, bmQ, bmB, bmP, ls, le, my_cuts, kMaxLocalMembers, open, cand);
            regular = cand && m >= 0;
            nm = regular ? (uint32_t)m : 0u;
        }
        uint32_t slots_total;
        const uint32_t slot0 = block_exclusive_scan(nm, scan_ws, slots_total);
        if (slots_total > (uint32_t)kSlots) {  // CTA-uniform, rare: keep the lines whose slots fit, redo the rest next round
            r = __syncthreads_count(active && slot0 + nm <= (uint32_t)kSlots);  // >= 1: one line holds <= kMaxLocalMembers members
            active = lt && tid < r;
        }
        bool fast = walk && regular && active;
        if (lt) {
            line_ls[tid] = ls;
            line_o0[tid] = o0;
            line_open[tid] = open;
            line_slot[tid] = slot0 | ((fast ? nm : 0u) << 16);
            line_bad[tid] = 0u;
            if (tid == r - 1) s_slots = slot0 + (fast ? nm : 0u);
        }
        if (fast) {
            for (uint32_t k = 0; k < nm; ++k) {
                cuts[slot0 + k] = my_cuts[k];
                slot_line[slot0 + k] = (uint8_t)tid;
            }
        }
        __syncthreads();
        const uint32_t nslots = s_slots;

        // ---- (4) one thread per member; numbers are only listed ----------------------------------------------------------------
        for (uint32_t sb = 0; sb < nslots; sb += (uint32_t)kThreads) {  // warp-uniform trip count: gf_member runs in lock step
            const uint32_t s = sb + (uint32_t)tid;
            const bool act = s < nslots;
            uint32_t l = 0;
            int a = 0, b = 0;
            if (act) {
                l = slot_line[s];
                const uint32_t k = s - (line_slot[l] & 0xFFFFu);
                a = k == 0u ? line_open[l] + 1 : (int)cuts[s - 1] + 1;
                b = (int)cuts[s];
            }
            int2 name = make_int2(0, 0);
            unsigned long long val = 0;
            uint32_t meta = 0;
            const bool good = gf_member(tile, bmQ, bmB, a, b, line_o0[l], line_ls[l], act, name, val, meta);
            if (act) {
                if (good) {
                    st_name[s] = name;
                    st_val[s] = val;
                    st_meta[s] = (uint8_t)meta;
                    if (meta == kGfNumber) {
                        // short tokens (levels, small integers) from the front of the list, long ones (timestamps, floats)
                        // from its end: lanes that run json_number side by side then loop about equally long
                        const bool lng = (int)((val >> 32) & 0xFFFFu) - (int)(val & 0xFFFFu) > 6;
                        if (lng) numlist[kSlots - 1 - (int)atomicAdd(&s_nlong, 1u)] = (uint16_t)s;
                        else numlist[atomicAdd(&s_nnum, 1u)] = (uint16_t)s;
                    }
                } else {
                    line_bad[l] = 1u;
                }
            }
        }
        __syncthreads();
        // ... and go through json_number side by side: every lane of these warps holds a number
        {
            const uint32_t nshort = s_nnum, nall = nshort + s_nlong;
            for (uint32_t q = (uint32_t)tid; q < nall; q += (uint32_t)kThreads) {
                const uint32_t s = q < nshort ? numlist[q] : numlist[kSlots - 1 - (int)(q - nshort)];
                unsigned long long val = 0;
                uint32_t meta = 0;
                if (gf_member_number(tile, st_val[s], val, meta)) {
                    st_val[s] = val;
                    st_meta[s] = (uint8_t)meta;
                } else {
                    line_bad[slot_line[s]] = 1u;
                }
            }
        }
        __syncthreads();

        // ---- (5) one thread per line: BTreeMap order, last duplicate wins, the per-key rules; rows over the line's slots -
        if (fast && line_bad[tid]) fast = false;
        const bool slow = walk && active && !fast;
        LineResult res;
        gelf_result_init(res);
        if (fast) {
            Members M;
            M.m = nm;
            M.spilled = false;
            for (uint32_t k = 0; k < nm; ++k) {
                M.name[k] = st_name[slot0 + k];
                M.val[k] = st_val[slot0 + k];
                M.meta[k] = st_meta[slot0 + k];
            }
            GelfAcc g;
            g.status = FG_ST_OK;
            g.flags = 0;
            g.kept = 0;
            g.have_ts = false;
            gf_finish(tile + ls, o0, M, res, g, stage, slot0);
            gelf_finalize(res, g);
        }
        if (bad_utf8) {
            res.status = FG_ES_INVALID_UTF8;
            res.n_entries = 0;
            res.full_o = 0;
        }
        const uint32_t my_n = (fast && res.status == FG_ST_OK) ? res.n_entries : 0u;
        uint32_t total;
        const uint32_t excl = block_exclusive_scan(my_n, scan_ws, total);
        uint32_t slow_total;
        const uint32_t slow_at = block_exclusive_scan(slow ? 1u : 0u, scan_ws, slow_total);
        if (lt) {
            line_slot[tid] = slot0 | (my_n << 16);
            line_dense[tid] = excl;
        }
        if (tid == 0 && total) s_ebase = atomicAdd(P.entry_counter, total);
        if (tid == 32 && slow_total) s_slow_base = atomicAdd(P.slow_count, slow_total);
        __syncthreads();
        if (slow) P.slow_list[s_slow_base + slow_at] = (uint32_t)i;
        uint32_t my_begin = 0;
        if (total) {  // CTA-uniform
            const uint32_t ebase = s_ebase;
            const bool ovf = (unsigned long long)ebase + total > (unsigned long long)P.entry_cap;
            if (!ovf) {
                if (my_n) my_begin = ebase + excl;
                for (uint32_t s = (uint32_t)tid; s < nslots; s += (uint32_t)kThreads) {
                    const uint32_t l = slot_line[s];
                    const uint32_t ls_n = line_slot[l];
                    const uint32_t k = s - (ls_n & 0xFFFFu);
                    if (k < (ls_n >> 16)) {
                        const uint32_t j = ebase + line_dense[l] + k;
                        sink.name[j] = st_name[s];
                        sink.val[j] = st_val[s];
                        sink.meta[j] = st_meta[s];
                    }
                }
            }
        }
        if (active && !slow) write_row(P, i, o0, res, my_begin, my_n);
        __syncthreads();  // tile, bitmap, slots and scan scratch are reused by the next round
        cur += r;
    }
}

// the exact parser over the listed lines: one thread per line straight from global memory, rows through the scratch table
__global__ void __launch_bounds__(128) post_gelf_kernel(const __grid_constant__ ParseParams P) {
    if (*P.bad_offsets) return;
    const uint32_t cnt = *P.slow_count;
    const uint32_t lane = threadIdx.x & 31u;
    const EntrySink sink = {P.entry_name, P.entry_val, P.entry_meta};
    const EntrySink tmp = {P.tmp_name, P.tmp_val, P.tmp_meta};
    const uint32_t stride = gridDim.x * 128u;
    for (uint32_t j0 = (blockIdx.x * 4u + (threadIdx.x >> 5)) * 32u; j0 < cnt; j0 += stride) {
        const uint32_t j = j0 + lane;
        const bool valid = j < cnt;
        int line = 0, o0 = 0, len = 0;
        if (valid) {
            line = (int)P.slow_list[j];
            o0 = P.offsets[line];
            len = P.offsets[line + 1] - o0;
            if (P.strip_eol && len > 0) {
                if (P.strip_eol == 2) {
                    if (P.bytes[o0 + len - 1] == 0) --len;
                } else if (P.bytes[o0 + len - 1] == '\n') {
                    --len;
                    if (len > 0 && P.bytes[o0 + len - 1] == '\r') --len;
                }
            }
        }
        LineResult res;
        const uint32_t sidx = (uint32_t)o0 / 3u;  // a top-level member needs >= 5 input bytes (`"":0,`)
        gelf_parse_line(P.bytes + o0, len, o0, sidx, valid, res, tmp);
        if (!valid) continue;
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
        write_row(P, line, o0, res, my_begin, my_n);
    }
}

}  // namespace

int parse_gelf_smem_bytes(int tile_bytes) {
    return tile_bytes + 3 * (tile_bytes / 32 + 4) * 4 + kCtrlWords * 4 + kGelfStageSlots * (8 + 8 + 2 + 2 + 1 + 1) + 16;
}

cudaError_t configure_parse_gelf(int max_tile_bytes) {
    {   // serde_json's POW10 table (visit_f64_from_parts): correctly rounded decimal literals, like rustc's
        static Pow10Table t;
        for (int k = 0; k <= 308; ++k) {
            char buf[16];
            snprintf(buf, sizeof buf, "1e%d", k);
            t.v[k] = strtod(buf, nullptr);
        }
        cudaError_t e1 = cudaMemcpyToSymbol(g_pow10, &t, sizeof t);  // this translation unit's copy: the one the GELF kernels read
        if (e1 != cudaSuccess) return e1;
    }
    return cudaFuncSetAttribute(parse_gelf_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, parse_gelf_smem_bytes(max_tile_bytes));
}

cudaError_t launch_parse_gelf(const ParseParams& p, cudaStream_t stream) {
    if (p.n <= 0) return cudaSuccess;
    if (p.tile_bytes <= 0 || p.tile_bytes > kGelfMaxTile || (p.tile_bytes & 511)) return cudaErrorInvalidValue;
    const int grid = (p.n + kLines - 1) / kLines;
    parse_gelf_kernel<<<grid, kThreads, parse_gelf_smem_bytes(p.tile_bytes), stream>>>(p);
    // the work list lives on the device (no host round trip): a fixed grid strides over it
    const int post = (int)min((long long)(p.n + 127) / 128, (long long)p.num_sms * 8);
    post_gelf_kernel<<<post, 128, 0, stream>>>(p);
    return cudaGetLastError();
}

}  // namespace fg
