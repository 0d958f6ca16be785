// emu_frame.cpp — the fused GELF encoder's output.framing arithmetic (fg_out_frame.cuh) compiled with g++ (TEST
// INFRASTRUCTURE, see cuda_shim.h): the syslen prefix writer, the framed / unframed record lengths and
// the frame the write pass stores around a record.
#define FG_HOST_EMU 1
#include <cstdint>

#include "../../flowgger_b200/csrc/fg_out_frame.cuh"

extern "C" {

int emu_syslen_prefix(unsigned long long len, uint8_t* out) { return fg::syslen_prefix(len, out); }
unsigned long long emu_framed_len(unsigned long long len, int framing) { return fg::framed_len(len, framing); }
unsigned long long emu_unframed_len(unsigned long long framed, int framing) { return fg::unframed_len(framed, framing); }
// the write pass of one record: its frame stored around its place, then its bytes where frame_record says
void emu_write_framed(const uint8_t* rec, unsigned long long len, int framing, uint8_t* out) {
    uint8_t* at = fg::frame_record(framing, fg::framed_len(len, framing), out);
    for (unsigned long long k = 0; k < len; ++k) at[k] = rec[k];
}

}  // extern "C"
