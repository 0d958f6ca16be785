// fg_rfc5424.cuh — one RFC5424 line -> Record fields, on device: the WIDE path (round-1 scanner).
//
// Since round 2 the hot path is fg_r5fast.cuh (structural bitmap + bit-walk over the shared-memory tile).  This file
// keeps the self-contained SWAR scanner that reads a line straight from global memory; post5424_kernel (wide_lines)
// (fg_parse5424.cu) runs it for the rare lines the fast path hands over: lines of 64 KiB or more (the compact rows
// hold u16 positions), lines longer than the staging tile, and lines whose side-table rows do not fit behind the
// cursor.  The block-scan primitives at the top are shared with the LTSV / GELF parsers.
//
// H100-native replacement for RFC5424Decoder::decode
// (flowgger src/flowgger/decoder/rfc5424_decoder.rs:18-49) and its helpers
// BOM::parse :63-71, parse_pri_version :74-92, rfc3339_to_unix :94-99,
// parse_data :127-161, parse_msg :163-172, parse_sd_data :174-242.
// The table rows carry the raw value span plus FG_EM_UNESCAPE; post5424_kernel (wide_lines) then rewrites
// those values (:105-125) into the batch arena.
//
// One thread owns one line.  SIMT discipline: the 32 lines of a
// warp advance in LOCK STEP through the same phases; every data-dependent loop
// is a warp-uniform `while (__any_sync(..))` whose body is predicated per lane,
// so lanes never skew into different code (without it the lanes of a warp
// ran one or two at a time).
// All 32 lanes of a warp MUST call rfc5424_parse_line (idle lanes with len = 0).
#pragma once
#include "fg_common.cuh"
#include "fg_kernels.cuh"
#include "fg_status.h"

namespace fg {

constexpr uint32_t kFullMask = 0xFFFFFFFFu;

struct LineResult {
    double ts;
    uint32_t status;
    uint32_t facility, severity, flags;
    // spans relative to the line start; off < 0 => None
    int host_o, host_l, app_o, app_l, proc_o, proc_l, mid_o, mid_l, msg_o, msg_l, full_o, full_l;
    uint32_t n_entries;  // SD headers + pairs of this line
};

// side-table columns (LTSV / GELF: provisional rows live in a scratch table indexed by the line's byte offset,
// see Format<>::scratch_index; RFC5424 wide path: final rows)
struct EntrySink {
    int2* name;
    unsigned long long* val;
    uint8_t* meta;
};


// --- 4-bytes-per-step scans over a line cursor ------------------------------------------------------
// `wp` = the line's bytes viewed as aligned 32-bit words (wp = p - a0, a0 = address of p & 3).  The word that
// holds byte i is wp[(a0 + i) >> 2]; bytes below the cursor are overwritten with 'A' (never a stop byte) so
// that the cheap zero-byte test (false positives only ABOVE a true positive) stays exact for the FIRST hit.
FG_DEV uint32_t swar_zero(uint32_t x) { return (x - 0x01010101u) & ~x & 0x80808080u; }  // 0x80 where byte == 0 (first hit exact)
FG_DEV uint32_t scan_word(const uint32_t* wp, uint32_t a0, int i, uint32_t& sh) {
    const uint32_t o = a0 + (uint32_t)i;
    sh = (o & 3u) * 8u;
    const uint32_t keep = 0xFFFFFFFFu << sh;
    return (wp[o >> 2] & keep) | (0x41414141u & ~keep);
}

// 16 bytes per step, for formats whose tokens are long (LTSV values, JSON strings): one 16-byte aligned load, an
// EXACT per-byte equality mask (0x80 where byte == pattern byte; no borrow artefacts, so hits below the cursor can
// simply be masked off), first hit at or after byte i.  Returns the new cursor: the hit position (`hit` = true) or
// the start of the next 16-byte block.  The block holding byte i is qp[(b0 + i) >> 4], b0 = address of p & 15.
FG_DEV uint32_t swar_eq(uint32_t w, uint32_t pat) {
    const uint32_t x = w ^ pat;
    return ~(((x & 0x7F7F7F7Fu) + 0x7F7F7F7Fu) | x | 0x7F7F7F7Fu);
}
// 0x80-per-byte flags of one word -> 4 bits in the top nibble (byte j -> bit 28 + j): the multiply moves bit 8j + 7 to
// bit 28 + j; every cross term lands on a distinct bit below 28, so nothing carries into the nibble
FG_DEV uint32_t swar_top_nibble(uint32_t z) { return z * 0x00204081u; }
// first flagged byte at or after the cursor (sh = cursor position inside the block), branch-free
FG_DEV int first_hit16(uint32_t z0, uint32_t z1, uint32_t z2, uint32_t z3, uint32_t sh, int i, bool& hit) {
    uint32_t m = (swar_top_nibble(z0) >> 28) | ((swar_top_nibble(z1) >> 24) & 0xF0u) | ((swar_top_nibble(z2) >> 20) & 0xF00u) |
                 ((swar_top_nibble(z3) >> 16) & 0xF000u);
    m &= 0xFFFFFFFFu << sh;
    hit = m != 0u;
    return i + (__ffs((int)(m | 0x10000u)) - 1) - (int)sh;  // no hit: the start of the next block
}
FG_DEV uint32_t swar_nibble(uint32_t z) { return swar_top_nibble(z) >> 28; }
template <bool TWO>
FG_DEV int scan_block16(const uint4* qp, uint32_t b0, int i, uint32_t pat1, uint32_t pat2, bool& hit) {
    const uint32_t o = b0 + (uint32_t)i;
    const uint4 v = qp[o >> 4];
    uint32_t z0 = swar_eq(v.x, pat1), z1 = swar_eq(v.y, pat1), z2 = swar_eq(v.z, pat1), z3 = swar_eq(v.w, pat1);
    if (TWO) {
        z0 |= swar_eq(v.x, pat2);
        z1 |= swar_eq(v.y, pat2);
        z2 |= swar_eq(v.z, pat2);
        z3 |= swar_eq(v.w, pat2);
    }
    return first_hit16(z0, z1, z2, z3, o & 15u, i, hit);
}
// JSON string body (serde_json read.rs ESCAPE table): '"', '\\' or a control byte (< 0x20)
FG_DEV uint32_t swar_json_stop(uint32_t w) { return swar_eq(w, 0x22222222u) | swar_eq(w, 0x5C5C5C5Cu) | swar_eq(w & 0xE0E0E0E0u, 0u); }
FG_DEV int scan_block16_json(const uint4* qp, uint32_t b0, int i, bool& hit) {
    const uint32_t o = b0 + (uint32_t)i;
    const uint4 v = qp[o >> 4];
    return first_hit16(swar_json_stop(v.x), swar_json_stop(v.y), swar_json_stop(v.z), swar_json_stop(v.w), o & 15u, i, hit);
}

// p: line bytes (global memory); len may be 0 for idle lanes.
// marks: this thread's column of a [6][stride] int array in shared memory (positions of the first six spaces).
// Side-table rows go to sink[sbase + k] when `emit` (the caller first runs a counting pass with emit = false, reserves
// r.n_entries rows and runs the line again).
template <int STRIDE>
FG_DEV void rfc5424_parse_line(bytes_t p, int len, int line_off, int* marks, LineResult& r, const EntrySink& sink, uint32_t sbase,
                               bool emit) {
    r.ts = 0.0;
    r.facility = 0xFFu;
    r.severity = 0xFFu;
    r.flags = 0;
    r.host_o = r.app_o = r.proc_o = r.mid_o = r.msg_o = r.full_o = -1;
    r.host_l = r.app_l = r.proc_l = r.mid_l = r.msg_l = r.full_l = 0;
    r.n_entries = 0;
    uint32_t status = FG_ST_OK;

    // ---- BOM::parse :63-71 ---------------------------------------------------------------------
    int b = 0;
    if (len >= 3 && p[0] == 0xEFu && p[1] == 0xBBu && p[2] == 0xBFu) b = 3;
    else if (!(len > 0 && p[0] == '<')) status = FG_E5_BOM;

    // ---- splitn(7, ' ') :23 — first six spaces, scanned a 16-byte block at a time -------------------
    int nsp = 0;
    {
        const uint8_t* q = p + b;
        const uint32_t s0 = (uint32_t)(size_t)q & 15u;
        const uint4* bq = (const uint4*)(q - s0);
        const int nblocks = (status == FG_ST_OK) ? (int)((s0 + (uint32_t)(len - b) + 15u) >> 4) : 0;
        int k = 0;
        bool active = nblocks > 0;
        while (__any_sync(kFullMask, active)) {
            if (active) {
                const uint4 v = bq[k];
                // one bit per byte == ' ' (exact SWAR equality, then the 0x80 flags of a word gathered into a nibble)
                uint32_t m = swar_nibble(swar_eq(v.x, 0x20202020u)) | (swar_nibble(swar_eq(v.y, 0x20202020u)) << 4) |
                             (swar_nibble(swar_eq(v.z, 0x20202020u)) << 8) | (swar_nibble(swar_eq(v.w, 0x20202020u)) << 12);
                if (k == 0) m &= 0xFFFFu << s0;
                while (m != 0 && nsp < 6) {
                    marks[nsp * STRIDE] = b + 16 * k + (__ffs((int)m) - 1) - (int)s0;
                    ++nsp;
                    m &= m - 1;
                }
                ++k;
                active = (k < nblocks) && (nsp < 6);
            }
        }
    }
    int sp0, sp1, sp2, sp3, sp4, sp5;
    {
        // marks past the end of the line come from the bytes after it in the last word: drop them
        int v;
        v = nsp > 0 ? marks[0 * STRIDE] : len; sp0 = v < len ? v : len;
        v = nsp > 1 ? marks[1 * STRIDE] : len; sp1 = v < len ? v : len;
        v = nsp > 2 ? marks[2 * STRIDE] : len; sp2 = v < len ? v : len;
        v = nsp > 3 ? marks[3 * STRIDE] : len; sp3 = v < len ? v : len;
        v = nsp > 4 ? marks[4 * STRIDE] : len; sp4 = v < len ? v : len;
        v = nsp > 5 ? marks[5 * STRIDE] : len; sp5 = v < len ? v : len;
        nsp = (sp0 < len) + (sp1 < len) + (sp2 < len) + (sp3 < len) + (sp4 < len) + (sp5 < len);
    }
    __syncwarp();

    // ---- parse_pri_version :74-92 on part0 = [b, sp0) --------------------------------------------
    if (status == FG_ST_OK) {
        const int e0 = sp0;
        if (!(b < e0 && p[b] == '<')) {
            status = FG_E5_PRI_BRACKETS;
        } else {
            int gt = b + 1;
            while (gt < e0 && p[gt] != '>') ++gt;
            uint32_t pri = 0;
            if (!parse_u8(p, b + 1, gt, pri)) status = FG_E5_INVALID_PRI;
            else if (gt >= e0) status = FG_E5_MISSING_VERSION;
            else if (!(e0 - gt == 2 && p[gt + 1] == '1')) status = FG_E5_UNSUPPORTED_VERSION;
            else {
                r.facility = pri >> 3;
                r.severity = pri & 7u;
            }
        }
    }
    __syncwarp();
    // ---- timestamp :25, :94-103 ---------------------------------------------------------------
    if (status == FG_ST_OK) {
        if (nsp < 1) status = FG_E5_MISSING_TS;
        else if (!parse_rfc3339(p, sp0 + 1, sp1, r.ts)) status = FG_E5_BAD_TS;
        else if (nsp < 6) status = FG_E5_MISSING_HOST + (uint32_t)(nsp - 1);  // :26-30 in order
    }
    __syncwarp();

    // ---- parse_data :127-161 on part6 = [sp5+1, len) -----------------------------------------------
    const int d = sp5 + 1;
    int msg_from = len;
    bool walk = false;
    if (status == FG_ST_OK) {
        if (d >= len) status = FG_E5_MISSING_MSG;  // :129
        else {
            const uint32_t c0 = p[d];
            if (c0 == '-') msg_from = d + 1;
            else if (c0 == '[') walk = true;
            else status = FG_E5_MALFORMED;  // :159
        }
    }
    {
        // Structured data, token-nested and in lock step: one outer iteration handles (per lane) either an
        // sd_id or one name="value" pair; the byte scans inside are tiny warp-uniform loops, so a warp pays
        // max-over-lanes of TOKEN lengths per step instead of a fat per-byte state machine.
        //   st_id : at the first byte of an sd_id (state ID of the reference walk, :175-177)
        //   !st_id: between params (state OUT: !in_name, name None, !in_value)
        uint32_t n = 1, pairs = 0, hdr = 0;
        const uint32_t a0 = (uint32_t)(size_t)p & 3u;
        const uint32_t* wp = (const uint32_t*)(p - a0);
        const uint32_t b0 = (uint32_t)(size_t)p & 15u;
        const uint4* qp = (const uint4*)(p - b0);
        int i = d + 1, elem_start = d + 1, id_end = 0;
        bool st_id = true;
        bool active = walk;
        // Inner scans are written as `lim`-bounded loops whose only loop-carried value is the cursor:
        // a lane that is not scanning has lim == i and falls through; nothing else is updated inside.
        while (__any_sync(kFullMask, active)) {
            // (A) sd_id: up to the first ' ' — 16 bytes per step (aligned block, hits before the cursor masked off)
            {
                const bool scan = active && st_id;
                const int lim = scan ? len : i;
                for (;;) {
                    bool more = false;
                    if (i < lim) {
                        bool hit;
                        i = scan_block16<false>(qp, b0, i, 0x20202020u, 0u, hit);  // stop on the space (may lie past len: checked below)
                        more = !hit;
                    }
                    if (!__any_sync(kFullMask, more)) break;
                }
                if (scan) {
                    if (i >= len) { active = false; status = FG_E5_MISSING_SD; }  // :177
                    else { id_end = i; ++i; st_id = false; }
                }
            }
            // (B) OUT: skip ' ' and stray '"' (:194, :232)
            {
                const int lim = active ? len : i;
                for (;;) {
                    uint32_t c = 0;
                    if (i < lim) c = p[i];
                    const bool more = (c == ' ') || (c == '"');
                    if (!__any_sync(kFullMask, more)) break;
                    i += more ? 1 : 0;
                }
                if (active && i >= len) { active = false; status = FG_E5_SD_NO_END; }  // :239
            }
            // classify the byte that ended (B)
            bool do_name = false;
            int name_start = 0, name_end = 0;
            if (active) {
                const uint32_t c = p[i];
                if (c == ']') {  // :197 end of this element, then :145-155
                    if (emit) {
                        const uint32_t e = sbase + hdr;
                        sink.name[e] = make_int2(line_off + elem_start, id_end - elem_start);
                        sink.val[e] = pairs;
                        sink.meta[e] = 7u;  // FG_TAG_SD_HEADER
                    }
                    if (i + 1 >= len) { active = false; status = FG_E5_MISSING_MSG; }  // :148
                    else {
                        const uint32_t c2 = p[i + 1];
                        if (c2 == '[') { elem_start = i + 2; i += 2; hdr = n++; pairs = 0; st_id = true; }
                        else if (c2 == ' ') { msg_from = i + 1; active = false; }
                        else { active = false; status = FG_E5_MALFORMED; }  // :154
                    }
                } else if (c >= 33u && c <= 126u && c != '=') {  // is_sd_name :188-192 ('"' and ']' excluded above)
                    do_name = true;
                    name_start = i;
                    ++i;
                } else {
                    active = false;
                    status = FG_E5_SD_FORMAT;  // :235
                }
            }
            // (C) NAME: name chars up to '=' (:205, :208) — 4 bytes per step; stop bytes: < 33, > 126, '"', '=', ']'
            {
                const int lim = do_name ? len : i;
                for (;;) {
                    bool more = false;
                    if (i < lim) {
                        uint32_t sh;
                        const uint32_t w = scan_word(wp, a0, i, sh);
                        const uint32_t z = ((w - 0x21212121u) & ~w & 0x80808080u)       // byte < 33
                                         | (((w + 0x01010101u) | w) & 0x80808080u)       // byte > 126
                                         | swar_zero(w ^ 0x22222222u) | swar_zero(w ^ 0x3D3D3D3Du) | swar_zero(w ^ 0x5D5D5D5Du);
                        if (z) i += (int)(((uint32_t)__ffs((int)z) - 1u - sh) >> 3);
                        else { i += 4 - (int)(sh >> 3); more = true; }
                    }
                    if (!__any_sync(kFullMask, more)) break;
                }
            }
            bool do_val = false;
            if (do_name) {
                if (i >= len) { active = false; status = FG_E5_SD_NO_END; }
                else if (p[i] != '=') { active = false; status = FG_E5_SD_FORMAT; }
                else {
                    name_end = i;
                    ++i;
                    if (i >= len) { active = false; status = FG_E5_SD_NO_END; }
                    else if (p[i] != '"') { active = false; status = FG_E5_SD_FORMAT; }  // :212 is the only arm
                    else { ++i; do_val = true; }
                }
            }
            // (D) VAL: up to the first unescaped '"' (:216, :217, :231) — 16 bytes per step
            uint32_t has_bs = 0;
            {
                const int lim = do_val ? len : i;
                for (;;) {
                    bool more = false;
                    if (i < lim) {
                        bool hit;
                        i = scan_block16<true>(qp, b0, i, 0x22222222u, 0x5C5C5C5Cu, hit);
                        more = !hit;
                        if (hit && i < lim && p[i] == '\\') { has_bs = 1u; i += 2; more = true; }  // escaped byte skipped
                    }
                    if (!__any_sync(kFullMask, more)) break;
                }
            }
            if (do_val) {
                if (i >= len) { active = false; status = FG_E5_SD_NO_END; }
                else {
                    if (emit) {
                        const uint32_t e = sbase + n;
                        sink.name[e] = make_int2(line_off + name_start, name_end - name_start);
                        sink.val[e] = (unsigned long long)(uint32_t)(line_off + name_end + 2) |
                                      ((unsigned long long)(uint32_t)(i - (name_end + 2)) << 32);
                        sink.meta[e] = (uint8_t)(has_bs ? 0x08u : 0u);  // FG_TAG_STRING | FG_EM_UNESCAPE
                    }
                    ++n;
                    ++pairs;
                    ++i;
                }
            }
        }
        if (walk && status == FG_ST_OK) r.n_entries = n;
    }

    // ---- parse_msg :163-172, Record assembly :32-47 ------------------------------------------------
    if (status == FG_ST_OK) {
        const int hi = trim_end(p, msg_from, len);
        const int lo = trim_start(p, msg_from, hi);
        if (hi > lo) {
            r.msg_o = lo;
            r.msg_l = hi - lo;
        }
        r.host_o = sp1 + 1;
        r.host_l = sp2 - sp1 - 1;
        r.app_o = sp2 + 1;
        r.app_l = sp3 - sp2 - 1;
        r.proc_o = sp3 + 1;
        r.proc_l = sp4 - sp3 - 1;
        r.mid_o = sp4 + 1;
        r.mid_l = sp5 - sp4 - 1;
        r.full_o = b;  // line.trim_end() of the BOM-stripped line :46
        r.full_l = trim_end(p, b, len) - b;
    }
    r.status = status;
    __syncwarp();
}

}  // namespace fg
