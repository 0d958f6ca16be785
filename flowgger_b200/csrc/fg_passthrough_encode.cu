// fg_passthrough_encode.cu — the passthrough encoder fused after the decoder on the device: Record -> header + full_msg
// (output.format = "passthrough").
//
// H100-native replacement for PassthroughEncoder::encode (flowgger src/flowgger/encoder/passthrough_encoder.rs:22-46).
// Record i is the header (output.syslog_prepend_timestamp, formatted by the caller once per call: fg_set_passthrough_prefix)
// followed by Record.full_msg, the bytes as they are.  full_msg is the span every record source of fg_encode_view.cuh
// already loads: the line after its BOM and trim_end for RFC5424, the trimmed line for RFC3164, the line as given for
// LTSV, and the unescaped full_message string for GELF.  A GELF Record without full_message is the encoder's error
// "Cannot output empty raw message" (FG_EP_NO_RAW): no record and no frame, like a decoder error.
//
// A record is at most two contiguous spans, so it is a gather-copy, not a text build:
//   size pass   one thread per line: header + full.len, framed.  Only a GELF full_message that holds JSON escapes
//               (FG_FLAG_FULL_ESC) is walked, with the decoder's unescape step, to count its unescaped bytes.
//   write pass  a warp copies its 32 records one at a time, all lanes on the same record (fg_warp_copy.cuh): header, then
//               body.  The lane of a record stores its frame first.  A body with JSON escapes is the one exception: after
//               the warp's copies, each lane unescapes its own such body into a WordSink (the LTSV encoder's byte loop).
// No tile is staged: each byte is read once, by a coalesced warp, so the kernels read global memory directly and
// launch with no dynamic shared memory.
#include "fg_encode_view.cuh"
#include "fg_ltsv_text.cuh"
#include "fg_out_frame.cuh"
#include "fg_warp_copy.cuh"

namespace fg {

namespace {

// the unescaped bytes of a JSON string body p[0, len) into `s`, four raw bytes at a time between escapes
template <class Sink>
__device__ __forceinline__ void unescape_span(const uint8_t* p, int len, bool mode2, Sink& s) {
    int k = 0;
    while (k < len) {
        uint32_t w = p[k];
        int n = 1;
        if (k + 4 <= len) {
            w |= ((uint32_t)p[k + 1] << 8) | ((uint32_t)p[k + 2] << 16) | ((uint32_t)p[k + 3] << 24);
            n = 4;
        }
        if (n == 1 || ltsv_eq4(w, 0x5C5C5C5Cu)) n = json_unescape_step(p, k, len, mode2, w);
        else k += n;
        s.push(w, n);
    }
    s.finish();
}

// Record.full_msg of a loaded row: its span, and whether it holds JSON escapes (GELF only).  false: the Record has none.
template <class Src>
__device__ __forceinline__ bool full_msg(const RecView& r, Span& body, bool& esc, bool& mode2) {
    body = r.full;
    esc = mode2 = false;
    if constexpr (Src::kGelf) {
        if (!r.full.p) return false;
        esc = (r.flags & kFullEsc) != 0u;
        mode2 = (r.flags & kNlRetry) != 0u;
    }
    return true;
}

template <class Src>
__global__ void __launch_bounds__(kEncLines) passthrough_size_kernel(const __grid_constant__ GelfEncodeParams P) {
    if (*P.bad_offsets) return;
    const int i = blockIdx.x * kEncLines + (int)threadIdx.x;
    if (i >= P.n) return;
    RecView r;
    Src::load(P, ByteSource{P.bytes, 0}, i, r);
    uint32_t st = Src::status(P, i);
    unsigned long long len = 0;
    Span body;
    bool esc, mode2;
    if (r.ok) {
        if (full_msg<Src>(r, body, esc, mode2)) {
            unsigned long long b = (unsigned)body.len;
            if (esc) {
                CountSink c;
                unescape_span(body.p, body.len, mode2, c);
                b = c.n;
            }
            len = framed_len((unsigned long long)(unsigned)P.n_static + b, P.out_framing);
        } else {
            st = FG_EP_NO_RAW;
        }
    }
    P.lens[i] = len;
    P.status[i] = (uint8_t)st;
    if constexpr (Src::kLtsv) P.ltsv_stop[i] = ltsv_stop(P, i);
}

template <class Src>
__global__ void __launch_bounds__(kEncLines) passthrough_write_kernel(const __grid_constant__ GelfEncodeParams P) {
    if (*P.bad_offsets) return;
    const int i = blockIdx.x * kEncLines + (int)threadIdx.x, lane = (int)(threadIdx.x & 31u);
    unsigned long long at = 0, len = 0;
    if (i < P.n) {
        at = P.base[0] + P.rel[i];
        len = P.lens[i];
        P.out_offsets[i] = (long long)at;
        if (i == P.n - 1) P.out_offsets[P.n] = (long long)(at + len);
    }
    // a rejected line has no record; an output buffer that overflowed is not written (the batch is redone)
    bool live = i < P.n && len != 0ull && at + len <= P.out_cap;
    Span body{nullptr, 0};
    bool esc = false, mode2 = false;
    uint8_t* dst = nullptr;
    if (live) {
        RecView r;
        Src::load(P, ByteSource{P.bytes, 0}, i, r);
        live = r.ok && full_msg<Src>(r, body, esc, mode2);
        if (live) dst = frame_record(P.out_framing, len, P.out + at);
    }
    // the warp's records one at a time: header, then the body unless it holds escapes
    const unsigned long long hdr = (unsigned)P.n_static;
    unsigned todo = __ballot_sync(0xFFFFFFFFu, live);
    while (todo) {
        const int j = __ffs((int)todo) - 1;
        todo &= todo - 1u;
        uint8_t* d = reinterpret_cast<uint8_t*>(__shfl_sync(0xFFFFFFFFu, reinterpret_cast<unsigned long long>(dst), j));
        const uint8_t* b = reinterpret_cast<const uint8_t*>(__shfl_sync(0xFFFFFFFFu, reinterpret_cast<unsigned long long>(body.p), j));
        const int bl = __shfl_sync(0xFFFFFFFFu, esc ? 0 : body.len, j);
        warp_copy(d, P.static_blob, hdr, lane);
        warp_copy(d + hdr, b, (unsigned)bl, lane);
    }
    if (live && esc) {  // GELF: this lane's full_message, unescaped
        WordSink s(dst + hdr);
        unescape_span(body.p, body.len, mode2, s);
    }
}

template <class Src>
cudaError_t configure_passthrough_src() {
    return configure_passes(passthrough_size_kernel<Src>, passthrough_write_kernel<Src>, 0);
}

template <class Src>
cudaError_t launch_passthrough_src(const GelfEncodeParams& p, void* d_scan_temp, size_t scan_temp_bytes, cudaStream_t stream) {
    GelfEncodeParams q = p;
    q.tile_bytes = 0;
    return launch_passes(passthrough_size_kernel<Src>, passthrough_write_kernel<Src>, q, d_scan_temp, scan_temp_bytes, stream);
}

}  // namespace

cudaError_t configure_passthrough_encode() {
    cudaError_t e = configure_passthrough_src<From5424>();
    if (e != cudaSuccess) return e;
    e = configure_passthrough_src<From3164>();
    if (e != cudaSuccess) return e;
    e = configure_passthrough_src<FromLtsv>();
    if (e != cudaSuccess) return e;
    return configure_passthrough_src<FromGelf>();
}

cudaError_t launch_passthrough_encode(int fmt, const GelfEncodeParams& p, void* d_scan_temp, size_t scan_temp_bytes, cudaStream_t stream) {
    if (p.n <= 0) return cudaSuccess;
    switch (fmt) {
        case 0: return launch_passthrough_src<From5424>(p, d_scan_temp, scan_temp_bytes, stream);
        case 1: return launch_passthrough_src<FromLtsv>(p, d_scan_temp, scan_temp_bytes, stream);
        case 2: return launch_passthrough_src<FromGelf>(p, d_scan_temp, scan_temp_bytes, stream);
        case 3: return launch_passthrough_src<From3164>(p, d_scan_temp, scan_temp_bytes, stream);
        default: return cudaErrorInvalidValue;
    }
}

}  // namespace fg
