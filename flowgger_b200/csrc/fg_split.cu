// fg_split.cu — device-side line framing + UTF-8 validation (SURVEY.md §8(f) N1).
//
// The same kernels frame NUL-delimited streams (NulSplitter, splitter/nul_splitter.rs:18-40: `BufRead::split(0)`, the
// delimiter is dropped, nothing else) — the delimiter byte is a launch parameter.
// Replaces the per-record work of LineSplitter::run (flowgger src/flowgger/splitter/line_splitter.rs:17-25):
// `BufRead::lines` (split at '\n', drop it and one preceding '\r', a last line without '\n' is still yielded) and the
// UTF-8 check of `String` (invalid line => "Invalid UTF-8 input", line skipped).  Input: a raw byte stream resident in
// HBM.  Output: int32 line-start offsets (line i = stream[offsets[i], offsets[i+1]) INCLUDING its terminator, which the
// parse kernels strip) and one invalid-UTF-8 flag per line.  These kernels are plain data-parallel byte scans (every
// byte read once per pass, 16-byte vector loads): two passes for the offsets (count, scan, fill) and one for UTF-8.
#include <cuda_runtime.h>
#include <stdint.h>

#include "fg_kernels.cuh"

namespace fg {

namespace {

constexpr int kSegBytes = 8192;   // one warp owns one segment
constexpr int kWarpsPerCta = 8;

// 0x80 in every byte == the record delimiter (exact for all bytes); pat = the delimiter in all four bytes
__device__ __forceinline__ uint32_t nl_flags(uint32_t w, uint32_t pat) {
    const uint32_t x = w ^ pat;
    return ~(((x & 0x7F7F7F7Fu) + 0x7F7F7F7Fu) | x | 0x7F7F7F7Fu);
}

// bytes beyond nbytes never equal the delimiter (the host pads the tail), so whole 16-byte loads are safe up to the padded end
__global__ void __launch_bounds__(kWarpsPerCta * 32) count_newlines_kernel(const uint8_t* __restrict__ bytes, long long nbytes,
                                                                            uint32_t* __restrict__ seg_counts, int seg0, int nseg, uint32_t pat) {
    const int seg = seg0 + blockIdx.x * kWarpsPerCta + (threadIdx.x >> 5);
    if (seg >= nseg) return;
    const uint32_t lane = threadIdx.x & 31u;
    const long long base = (long long)seg * kSegBytes;
    uint32_t cnt = 0;
#pragma unroll 4
    for (int row = 0; row < kSegBytes / 512; ++row) {
        const long long pos = base + row * 512 + lane * 16;
        if (pos < nbytes) {
            const uint4 v = *reinterpret_cast<const uint4*>(bytes + pos);
            cnt += __popc(nl_flags(v.x, pat)) + __popc(nl_flags(v.y, pat)) + __popc(nl_flags(v.z, pat)) + __popc(nl_flags(v.w, pat));
        }
    }
    cnt = __reduce_add_sync(0xFFFFFFFFu, cnt);
    if (lane == 0) seg_counts[seg] = cnt;
}

// single CTA: exclusive scan of the counts of segments [seg0, seg1) on top of the running newline count `*run`
// (chunk-pipelined framing: chunk k is scanned as soon as its bytes are resident).  Publishes the cumulative newline
// count after this chunk; the last chunk also settles the line count and the end offset of an unterminated last line.
__global__ void __launch_bounds__(1024) scan_segments_kernel(uint32_t* __restrict__ seg_counts, int seg0, int seg1, uint32_t* __restrict__ run,
                                                             int32_t* __restrict__ cum_out, int is_last, const uint8_t* __restrict__ bytes,
                                                             long long nbytes, int32_t* __restrict__ offsets, int32_t* __restrict__ n_lines,
                                                             int max_lines, uint32_t delim) {
    __shared__ uint32_t part[1024];
    const int t = threadIdx.x;
    const int nseg = seg1 - seg0;
    const int per = (nseg + 1023) / 1024;
    const int lo = seg0 + t * per, hi = min(seg1, lo + per);
    uint32_t s = 0;
    for (int k = lo; k < hi; ++k) s += seg_counts[k];
    part[t] = s;
    __syncthreads();
    for (int d = 1; d < 1024; d <<= 1) {
        const uint32_t v = t >= d ? part[t - d] : 0u;
        __syncthreads();
        part[t] += v;
        __syncthreads();
    }
    const uint32_t before = *run;
    uint32_t r = before + part[t] - s;  // exclusive prefix of this thread's range
    for (int k = lo; k < hi; ++k) {
        const uint32_t c = seg_counts[k];
        seg_counts[k] = r;
        r += c;
    }
    __syncthreads();
    if (t == 1023) {
        const unsigned long long newlines = (unsigned long long)before + part[1023];
        *run = (uint32_t)newlines;
        // records so far: bytes follow a chunk that is not the last, so one more record is open after it; after the last
        // chunk only an unterminated last record counts (BufRead::lines / split yield it), a terminated one has no successor
        const bool tail = is_last && nbytes > 0 && bytes[nbytes - 1] != delim;
        const unsigned long long n = newlines + (is_last ? (tail ? 1ull : 0ull) : 1ull);
        const bool over = n > (unsigned long long)max_lines;
        *cum_out = over ? -1 : (int32_t)newlines;
        if (seg0 == 0) offsets[0] = 0;
        if (is_last) {
            *n_lines = over ? -1 : (int32_t)n;
            if (!over && tail) offsets[n] = (int32_t)nbytes;
        }
    }
}

__global__ void __launch_bounds__(kWarpsPerCta * 32) fill_offsets_kernel(const uint8_t* __restrict__ bytes, long long nbytes,
                                                                          const uint32_t* __restrict__ seg_base, int seg0, int nseg,
                                                                          int32_t* __restrict__ offsets, int max_lines, uint32_t pat) {
    const int seg = seg0 + blockIdx.x * kWarpsPerCta + (threadIdx.x >> 5);
    if (seg >= nseg) return;
    const uint32_t lane = threadIdx.x & 31u;
    const long long base = (long long)seg * kSegBytes;
    uint32_t run = seg_base[seg];  // newlines before this segment
    for (int row = 0; row < kSegBytes / 512; ++row) {
        const long long pos = base + row * 512 + lane * 16;
        uint32_t z[4] = {0u, 0u, 0u, 0u};
        if (pos < nbytes) {
            const uint4 v = *reinterpret_cast<const uint4*>(bytes + pos);
            z[0] = nl_flags(v.x, pat); z[1] = nl_flags(v.y, pat); z[2] = nl_flags(v.z, pat); z[3] = nl_flags(v.w, pat);
        }
        const uint32_t c = __popc(z[0]) + __popc(z[1]) + __popc(z[2]) + __popc(z[3]);
        uint32_t inc = c;  // inclusive warp scan
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
            const uint32_t y = __shfl_up_sync(0xFFFFFFFFu, inc, d);
            if (lane >= (uint32_t)d) inc += y;
        }
        uint32_t k = run + inc - c;  // rank of this lane's first newline
#pragma unroll
        for (int wI = 0; wI < 4; ++wI) {
            uint32_t f = z[wI];
            while (f) {
                const int b = (__ffs((int)f) - 1) >> 3;
                if (k + 1 <= (uint32_t)max_lines) offsets[k + 1] = (int32_t)(pos + wI * 4 + b + 1);  // the next line starts after this '\n'
                ++k;
                f &= f - 1;
            }
        }
        run += __shfl_sync(0xFFFFFFFFu, inc, 31);
    }
}

// core::str::from_utf8 acceptance, data-parallel: every thread owns 16 bytes, validates the sequences that START in
// its chunk (reading up to 3 bytes beyond it) and checks that every continuation byte in its chunk is claimed by a
// lead byte at most 3 positions back.  Chunks of pure ASCII (the common case) cost four compares.
__device__ __forceinline__ int utf8_need(uint32_t c) {  // continuation bytes a lead byte announces; -1 = invalid lead
    if (c < 0x80u) return 0;
    if (c >= 0xC2u && c <= 0xDFu) return 1;
    if (c >= 0xE0u && c <= 0xEFu) return 2;
    if (c >= 0xF0u && c <= 0xF4u) return 3;
    return -1;  // 0x80..0xC1 (continuation or overlong lead), 0xF5..0xFF
}

// Validates the byte positions [v0, v1) (16-byte aligned bounds); everything it reads (up to 3 bytes past v1) must be
// resident, so the chunk-pipelined caller lags the validated window 16 bytes behind the uploaded bytes.  `known` = number of
// newlines found so far: lines 0 .. known (the last one possibly still open) have valid start offsets.
__global__ void __launch_bounds__(256) validate_utf8_kernel(const uint8_t* __restrict__ bytes, long long nbytes, long long v0, long long v1,
                                                            const int32_t* __restrict__ offsets, const int32_t* __restrict__ known,
                                                            uint8_t* __restrict__ invalid) {
    const int kn = *known;
    if (kn < 0) return;
    const int n = kn + 1;
    const long long pos = v0 + ((long long)blockIdx.x * blockDim.x + threadIdx.x) * 16;
    if (pos >= v1 || pos >= nbytes) return;
    const uint4 v = *reinterpret_cast<const uint4*>(bytes + pos);
    if (((v.x | v.y | v.z | v.w) & 0x80808080u) == 0u) return;  // ASCII only
    // an error flags the line that holds the offending byte (several lines may meet inside one chunk)
    auto flag = [&](long long bad) {
        int lo = 0, hi = n;  // offsets[lo] <= bad < offsets[hi]
        while (hi - lo > 1) {
            const int mid = (lo + hi) >> 1;
            if ((long long)offsets[mid] <= bad) lo = mid;
            else hi = mid;
        }
        invalid[lo] = 1;
    };
    long long end = pos + 16 < nbytes ? pos + 16 : nbytes;
    if (end > v1) end = v1;
    for (long long q = pos; q < end; ++q) {
        const uint32_t c = bytes[q];
        if (c < 0x80u) continue;
        if ((c & 0xC0u) == 0x80u) {
            // continuation byte: some lead within the 3 previous bytes must cover it
            bool claimed = false;
            for (int back = 1; back <= 3 && q - back >= 0; ++back) {
                const uint32_t l = bytes[q - back];
                if ((l & 0xC0u) == 0x80u) continue;  // another continuation byte: keep looking
                claimed = utf8_need(l) >= back;
                break;
            }
            if (!claimed) flag(q);
            continue;
        }
        const int need = utf8_need(c);
        if (need < 0) { flag(q); continue; }
        // continuation bytes (bytes past the end of the stream read as 0 and fail the check)
        uint32_t b1 = q + 1 < nbytes ? bytes[q + 1] : 0u;
        bool ok = (b1 & 0xC0u) == 0x80u;
        if (c == 0xE0u) ok = ok && b1 >= 0xA0u;             // overlong 3-byte
        else if (c == 0xEDu) ok = ok && b1 <= 0x9Fu;        // UTF-16 surrogates
        else if (c == 0xF0u) ok = ok && b1 >= 0x90u;        // overlong 4-byte
        else if (c == 0xF4u) ok = ok && b1 <= 0x8Fu;        // > U+10FFFF
        for (int k = 2; k <= need && ok; ++k) {
            const uint32_t bk = q + k < nbytes ? bytes[q + k] : 0u;
            ok = (bk & 0xC0u) == 0x80u;
        }
        if (!ok) flag(q);
    }
}

}  // namespace

// Framing + validation of the bytes [c0, c1) (c0 a multiple of the segment size) of a stream of nbytes bytes whose bytes
// [0, c1) are resident.  `d_run` carries the newline count across chunks, d_cum[k] receives the count after this chunk.
cudaError_t launch_split_chunk(const uint8_t* d_bytes, long long nbytes, long long c0, long long c1, int is_last, uint32_t* d_seg,
                               uint32_t* d_run, int32_t* d_cum_k, int32_t* d_offsets, int32_t* d_n_lines, int max_lines,
                               uint8_t* d_invalid, int delim, cudaStream_t stream) {
    const uint32_t pat = (uint32_t)(delim & 0xFF) * 0x01010101u;
    const int seg0 = (int)(c0 / kSegBytes), seg1 = (int)((c1 + kSegBytes - 1) / kSegBytes);
    const int grid = (seg1 - seg0 + kWarpsPerCta - 1) / kWarpsPerCta;
    if (seg1 > seg0) count_newlines_kernel<<<grid, kWarpsPerCta * 32, 0, stream>>>(d_bytes, nbytes < c1 ? nbytes : c1, d_seg, seg0, seg1, pat);
    scan_segments_kernel<<<1, 1024, 0, stream>>>(d_seg, seg0, seg1, d_run, d_cum_k, is_last, d_bytes, nbytes, d_offsets, d_n_lines, max_lines, (uint32_t)(delim & 0xFF));
    if (seg1 > seg0) {
        fill_offsets_kernel<<<grid, kWarpsPerCta * 32, 0, stream>>>(d_bytes, nbytes < c1 ? nbytes : c1, d_seg, seg0, seg1, d_offsets, max_lines, pat);
        // validated window lags 16 bytes behind the resident bytes (sequences read up to 3 bytes ahead), except at the end
        const long long v0 = c0 >= 16 ? c0 - 16 : 0, v1 = is_last ? ((nbytes + 15) & ~15LL) : c1 - 16;
        if (v1 > v0) {
            const long long chunks = (v1 - v0 + 15) / 16;
            validate_utf8_kernel<<<(unsigned)((chunks + 255) / 256), 256, 0, stream>>>(d_bytes, nbytes, v0, v1, d_offsets, d_cum_k, d_invalid);
        }
    }
    return cudaGetLastError();
}

int split_segments(long long nbytes) { return (int)((nbytes + kSegBytes - 1) / kSegBytes); }

}  // namespace fg
