// emu_capnp.cpp — CPU emulation of the fused Cap'n Proto encoder's layout (TEST INFRASTRUCTURE, see cuda_shim.h).
//
// Compiles the product's allocator and pointer words (fg_capnp_layout.cuh) with g++ and places one message's objects
// the way capnp_size_kernel / capnp_write_kernel (fg_capnp_encode.cu) do: each object is placed from the segment that
// holds its pointer, and its pointer (and landing pad) words are computed from where it went.
#define FG_HOST_EMU 1
#include <cstdint>

#include "cuda_shim.h"
#include "../../flowgger_b200/csrc/fg_capnp_layout.cuh"

extern "C" {

// n objects in allocation order.  type: 0 the Record (value unused), 1 a text of `value` bytes, 2 a Pair list of `value`
// pairs.  Its pointer: container[t] = -1 -> word ptr_off[t] of segment 0, else word pos[container] + ptr_off[t] of the
// container's segment.  Out per object: seg, pos, pad (-1: none), the pointer word and the landing pad word (0: none);
// out: the segment table words (*ntable) and the message bytes.  Returns 1 when the allocator refuses the record.
int emu_capnp_layout(int n, const int32_t* type, const uint32_t* value, const int32_t* container, const uint32_t* ptr_off, int32_t* seg,
                     uint32_t* pos, int32_t* pad, unsigned long long* ptr_word, unsigned long long* pad_word, unsigned long long* table,
                     int32_t* ntable, unsigned long long* bytes) {
    fg::CapAlloc A;
    A.init();
    for (int t = 0; t < n; ++t) {
        const int c = container[t];
        const int ps = c < 0 ? 0 : seg[c];
        const uint32_t pw = c < 0 ? ptr_off[t] : pos[c] + ptr_off[t];
        uint32_t words, kind, hi;
        if (type[t] == 0) {
            words = fg::kCapRootWords;
            kind = 0;
            hi = fg::cap_struct_hi(2, 9);
        } else if (type[t] == 1) {
            words = fg::cap_text_words(value[t]);
            kind = 1;
            hi = fg::cap_text_hi(value[t]);
        } else {
            words = 1u + 4u * value[t];
            kind = 1;
            hi = fg::cap_pairs_hi(value[t]);
        }
        const fg::CapPlace pl = A.place(ps, words);
        seg[t] = pl.seg;
        pos[t] = pl.pos;
        pad[t] = pl.pad;
        ptr_word[t] = fg::cap_pointer(ps, pw, pl, kind, hi);
        pad_word[t] = pl.pad >= 0 ? fg::cap_pad_word(kind, hi) : 0ull;
    }
    *ntable = A.table_words();
    for (int k = 0; k < A.table_words(); ++k) table[k] = A.table_word(k);
    *bytes = A.bytes();
    return A.bad ? 1 : 0;
}

unsigned long long emu_capnp_pairs_tag(uint32_t n) { return fg::cap_pairs_tag(n); }

}  // extern "C"
