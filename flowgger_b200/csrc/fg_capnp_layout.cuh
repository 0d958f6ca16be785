// fg_capnp_layout.cuh — where capnp-rust 0.14 puts each object of a message, and the pointer words that reach it.
//
// The fused Cap'n Proto encoder (fg_capnp_encode.cu) builds what Builder::new_default() + build_record +
// serialize::write_message build (encoder/capnp_encoder.rs:36-109).  A message is a list of segments; objects are
// allocated one after the other, and each is first tried in the segment that holds its pointer.  When it does not fit,
// it takes n + 1 words — a landing pad, then the object — in the first segment with room, in order 0..k
// (allocate_anywhere), or else in a new segment of max(n + 1, next_size) words, next_size starting at 2048 and growing
// by the size of each new segment (HeapAllocator, GrowHeuristically); the pointer becomes a far pointer to the pad.
// Segment 0 has 1024 words: the root pointer at word 0, then the objects.  Host and device code (the CPU tests compile
// it with g++).
#pragma once
#include <cstdint>

namespace fg {

constexpr uint32_t kCapSeg0Words = 1024;
constexpr uint32_t kCapNextWords = 2048;
constexpr int kCapMaxSegs = 24;                 // 1024 * 2^23 words: far beyond any record a line can give
constexpr uint32_t kCapMaxWords = 1u << 29;     // list lengths, and pointer offsets within a segment, stop here
constexpr uint32_t kCapRootWords = 11;          // Record: 2 data words, 9 pointers

// An object's place: segment, first word, and the word of its landing pad (-1: reached directly from its pointer)
struct CapPlace {
    int seg;
    uint32_t pos;
    int32_t pad;
};

struct CapAlloc {
    uint32_t size[kCapMaxSegs], used[kCapMaxSegs];
    int nseg;
    uint32_t next;
    bool bad;  // more segments than kCapMaxSegs, or a segment past kCapMaxWords: the record is refused
    __host__ __device__ __forceinline__ void init() {
        nseg = 1;
        size[0] = kCapSeg0Words;
        used[0] = 1;  // the root pointer
        next = kCapNextWords;
        bad = false;
    }
    // n words for an object whose pointer lies in segment p
    __host__ __device__ __forceinline__ CapPlace place(int p, uint32_t n) {
        if (n <= size[p] - used[p]) {
            const uint32_t at = used[p];
            used[p] += n;
            return CapPlace{p, at, -1};
        }
        const uint32_t m = n + 1;
        int s = 0;
        while (s < nseg && m > size[s] - used[s]) ++s;
        if (s == nseg) {
            if (nseg == kCapMaxSegs) {
                bad = true;
                s = nseg - 1;
                used[s] = 0;
            } else {
                const uint32_t sz = m > next ? m : next;
                size[s] = sz;
                used[s] = 0;
                next += sz;
                ++nseg;
                if (sz > kCapMaxWords) bad = true;
            }
        }
        const uint32_t at = used[s];
        used[s] += m;
        return CapPlace{s, at + 1, (int32_t)at};
    }
    // bytes of the message: the segment table (u32 count - 1, u32 words per segment, padded to 8 bytes), then the words
    __host__ __device__ __forceinline__ unsigned long long bytes() const {
        unsigned long long w = 0;
        for (int s = 0; s < nseg; ++s) w += used[s];
        return 8ull * ((unsigned)nseg / 2u + 1u) + 8ull * w;
    }
    // word k of the segment table
    __host__ __device__ __forceinline__ unsigned long long table_word(int k) const {
        const int a = 2 * k - 1, b = 2 * k;  // u32 slot 2k holds segment 2k - 1 (slot 0: the count - 1)
        const unsigned long long lo = k == 0 ? (unsigned long long)(nseg - 1) : used[a];
        const unsigned long long hi = b < nseg ? used[b] : 0ull;
        return lo | (hi << 32);
    }
    __host__ __device__ __forceinline__ int table_words() const { return nseg / 2 + 1; }
};

// the words of a text of `len` bytes: its NUL, rounded up to whole words
__host__ __device__ __forceinline__ uint32_t cap_text_words(uint32_t len) { return (len + 8u) >> 3; }

// the upper half of a pointer: a struct's data words and pointers, or a list's element size and count
__host__ __device__ __forceinline__ uint32_t cap_struct_hi(uint32_t data, uint32_t ptrs) { return data | (ptrs << 16); }
__host__ __device__ __forceinline__ uint32_t cap_text_hi(uint32_t len) { return 2u | ((len + 1u) << 3); }         // bytes
__host__ __device__ __forceinline__ uint32_t cap_pairs_hi(uint32_t n) { return 7u | ((4u * n) << 3); }           // composite
__host__ __device__ __forceinline__ unsigned long long cap_pairs_tag(uint32_t n) {                               // its tag
    return (unsigned long long)(n << 2) | ((unsigned long long)cap_struct_hi(2, 2) << 32);
}

// The pointer at word w of segment p to an object placed at `pl`; kind 0 = struct, 1 = list; hi = the upper half.  A far
// pointer names the landing pad, which is the pointer with offset 0 (cap_pad_word).
__host__ __device__ __forceinline__ unsigned long long cap_pointer(int p, uint32_t w, const CapPlace& pl, uint32_t kind, uint32_t hi) {
    if (pl.pad >= 0) return 2ull | ((unsigned long long)(uint32_t)pl.pad << 3) | ((unsigned long long)(uint32_t)pl.seg << 32);
    const uint32_t off = (uint32_t)((int32_t)(pl.pos - w - 1u) * 4);
    return (unsigned long long)(off | kind) | ((unsigned long long)hi << 32);
}
__host__ __device__ __forceinline__ unsigned long long cap_pad_word(uint32_t kind, uint32_t hi) {
    return (unsigned long long)kind | ((unsigned long long)hi << 32);
}

}  // namespace fg
