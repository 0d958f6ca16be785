// fg_parse3164.cu — the RFC3164 decoder on sm_90a (SURVEY.md §8(f) N3): bytes -> row columns (+ re-joined messages).
//
//   parse3164_kernel   one CTA = 64 consecutive lines, 64 threads.
//     (1) thread 0 issues ONE TMA bulk copy (cp.async.bulk, SASS UBLKCP) of the lines' contiguous byte span into the
//         shared-memory tile: HBM is read once, coalesced, without per-thread global loads;
//     (2) one thread per line runs r3164_parse_line (fg_rfc3164.cuh) over its bytes in the tile.  A line is an independent
//         unit with a fixed-size result, so there is no CTA phase after the tile wait: the threads neither vote nor
//         exchange data, and the row columns are written by consecutive threads (coalesced);
//     (3) a message whose tokens are not separated by single spaces is re-joined into the arena (one atomic per such line).
//   Lines of the CTA that do not fit the tile (far longer than the batch mean) are parsed straight from global memory by
//   their own thread.  RFC3164 records have no structured data: the side table stays empty.
#include "fg_kernels.cuh"

#include "fg_common.cuh"
#define FG_R3164_WALKERS 1
#include "fg_rfc3164.cuh"
#include "fg_status.h"
#include "fg_tma.cuh"

namespace fg {

namespace {

constexpr int kLines = kR3164LinesPerCta;
static_assert(kLines % 32 == 0, "r3164_parse_lockstep is called by whole warps");

__global__ void __launch_bounds__(kLines, kR3164CtasPerSm) parse3164_kernel(const __grid_constant__ ParseParams P) {
    extern __shared__ __align__(128) uint8_t tile[];
    __shared__ __align__(8) uint64_t mbar;

    if (*P.bad_offsets) return;  // CTA-uniform
    const int tid = threadIdx.x;
    const int first = blockIdx.x * kLines;
    const int last = min(P.n, first + kLines);
    const int i = first + tid;
    if (tid == 0) mbar_init(&mbar, 1);
    int o0 = 0, o1 = 0;
    if (i < last) {
        o0 = __ldg(P.offsets + i);
        o1 = __ldg(P.offsets + i + 1);
    }
    const int base = __ldg(P.offsets + first) & ~15;
    const bool fits = i < last && o1 - base <= P.tile_bytes;  // offsets are monotone: a prefix of the CTA's lines
    const int r = __syncthreads_count(fits);                  // (also publishes the mbarrier initialisation)
    if (r > 0) {
        if (tid == 0) {
            const int oend = __ldg(P.offsets + first + r);
            const uint32_t nbytes = (uint32_t)((oend - base) + 15) & ~15u;  // <= tile_bytes (a multiple of 512); the input buffer is padded
            mbar_expect_tx(&mbar, nbytes);
            bulk_g2s(tile, P.bytes + base, nbytes, &mbar);
        }
        mbar_wait(&mbar, 0u);
    }
    const bool have = i < last;
    const uint8_t* lp = fits ? tile + (o0 - base) : P.bytes + o0;
    int len = o1 - o0;
    bool bad_utf8 = false;
    if (have && P.strip_eol && len > 0) {
        // BufRead::lines drops the '\n' and one '\r' before it (line_splitter.rs:17); BufRead::split(0) only the NUL
        // (nul_splitter.rs:18); a record that is not UTF-8 is reported and skipped (:22-25)
        if (P.strip_eol == 2) {
            if (lp[len - 1] == 0) --len;
        } else if (lp[len - 1] == '\n') {
            --len;
            if (len > 0 && lp[len - 1] == '\r') --len;
        }
        bad_utf8 = P.line_invalid != nullptr && P.line_invalid[i] != 0;
    }
    R3Out res;
#if FG_R3_LOCKSTEP
    // every lane of the warp walks the same phases (lanes without a line idle): see fg_rfc3164.cuh
    r3164_parse_lockstep(lp, len, have && !bad_utf8, P.r3164, res);
    if (!have) return;
    if (bad_utf8) res.status = FG_ES_INVALID_UTF8;
#else
    if (!have) return;
    if (bad_utf8) {
        res.status = FG_ES_INVALID_UTF8;
        res.facility = res.severity = 0xFFu;
        res.flags = 0u;
        res.ts = 0.0;
    } else if (fits) {
        r3164_parse_line(tile + (o0 - base), len, P.r3164, res);  // shared-memory loads (LDS) on the common path
    } else {
        r3164_parse_line(P.bytes + o0, len, P.r3164, res);
    }
#endif
    const bool ok = res.status == FG_ST_OK;
    P.ts[i] = ok ? res.ts : 0.0;
    P.meta[i] = res.status | (res.facility << 8) | (res.severity << 16) | (res.flags << 24);
    P.host[i] = ok ? make_int2(o0 + res.host_o, res.host_l) : make_int2(-1, 0);
    P.msg[i] = ok ? make_int2((res.flags & kR3FlagMsgArena) ? res.msg_o : o0 + res.msg_o, res.msg_l) : make_int2(-1, 0);
    P.full[i] = ok ? make_int2(o0, res.full_l) : make_int2(-1, 0);
    P.sd[i] = make_int2(0, 0);
}

int smem_bytes(int tile_bytes) { return tile_bytes + 16; }

}  // namespace

cudaError_t configure_parse3164(int max_tile_bytes) {
    return cudaFuncSetAttribute(parse3164_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_bytes(max_tile_bytes));
}

cudaError_t launch_parse3164(const ParseParams& p, cudaStream_t stream) {
    if (p.n <= 0) return cudaSuccess;
    if (p.tile_bytes <= 0 || p.tile_bytes > kR3164MaxTile || (p.tile_bytes & 511)) return cudaErrorInvalidValue;
    const int grid = (p.n + kLines - 1) / kLines;
    parse3164_kernel<<<grid, kLines, smem_bytes(p.tile_bytes), stream>>>(p);
    return cudaGetLastError();
}

}  // namespace fg
