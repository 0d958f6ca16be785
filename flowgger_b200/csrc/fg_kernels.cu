// fg_kernels.cu — configuration and dispatch of the batched parse kernels (sm_90a).
//
// RFC5424, LTSV and GELF run on the same pipeline (DESIGN.md §3), each in its own file; RFC3164 shares the staging only:
//   RFC5424  fg_parse5424.cu   parse5424_kernel + post5424_kernel
//   LTSV     fg_parse_ltsv.cu  parse_ltsv_kernel
//   GELF     fg_parse_gelf.cu  parse_gelf_kernel + post_gelf_kernel
//   RFC3164  fg_parse3164.cu   parse3164_kernel (tile + one thread per line, no bitmap stage)
// one CTA = 64 consecutive lines whose contiguous byte span is staged in shared memory by ONE TMA bulk copy
// (cp.async.bulk, SASS UBLKCP); all threads sweep the tile into structural bitmaps; one thread per line walks its tokens over
// the bitmaps in lock step; side-table rows are staged in shared memory, placed by a CTA scan + one global atomic and
// copied out coalesced.
#include "fg_kernels.cuh"

#include "fg_common.cuh"
#include "fg_status.h"

namespace fg {

cudaError_t configure_kernels(int max_tile5424) {
    cudaError_t e = configure_parse5424(max_tile5424);
    if (e != cudaSuccess) return e;
    e = configure_gelf_encode(max_tile5424);
    if (e != cudaSuccess) return e;
    e = configure_ltsv_encode(max_tile5424);
    if (e != cudaSuccess) return e;
    e = configure_capnp_encode(max_tile5424);
    if (e != cudaSuccess) return e;
    e = configure_passthrough_encode();
    if (e != cudaSuccess) return e;
    e = configure_parse_ltsv(kLtsvMaxTile);
    if (e != cudaSuccess) return e;
    e = configure_parse_gelf(kGelfMaxTile);
    if (e != cudaSuccess) return e;
    return configure_parse3164(kR3164MaxTile);
}

__global__ void __launch_bounds__(256) check_offsets_kernel(const int32_t* __restrict__ offsets, int n, long long max_bytes,
                                                           uint32_t* __restrict__ flag) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i > n) return;
    const int a = offsets[i];
    bool bad = a < 0 || (long long)a > max_bytes;
    if (i < n) bad = bad || offsets[i + 1] < a;
    if (bad) atomicOr(flag, 1u);
}

cudaError_t launch_check_offsets(const int32_t* d_offsets, int n, long long max_bytes, uint32_t* d_flag, cudaStream_t stream) {
    if (n <= 0) return cudaSuccess;
    check_offsets_kernel<<<(n + 1 + 255) / 256, 256, 0, stream>>>(d_offsets, n, max_bytes, d_flag);
    return cudaGetLastError();
}

cudaError_t launch_parse(int fmt, const ParseParams& p, cudaStream_t stream) {
    switch (fmt) {
        case 1: return launch_parse_ltsv(p, stream);
        case 2: return launch_parse_gelf(p, stream);
        case 3: return launch_parse3164(p, stream);
        default: return cudaErrorInvalidValue;
    }
}

const char* kernel_build_info() {
    return "flowgger_b200 parse kernels: sm_90a, structural bitmaps + bit-walk over TMA-bulk-staged CTA tiles, "
           "kernels=[parse5424_kernel, post5424_kernel, gelf_size_kernel, gelf_write_kernel, ltsv_size_kernel, ltsv_write_kernel, capnp_size_kernel, capnp_write_kernel, passthrough_size_kernel, passthrough_write_kernel, parse_ltsv_kernel, parse_gelf_kernel, post_gelf_kernel, parse3164_kernel]";
}

}  // namespace fg
