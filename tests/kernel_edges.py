"""Batches that sit on the capacity limits of the device kernels (test infrastructure, pure Python, no GPU).

Every parse kernel stages a CTA's lines in a shared-memory tile, cuts a round short when the next line or its parts do
not fit, sends a line that does not fit alone to another path, and packs positions into 16 bits.  The builders below put
lines one byte below, on and one byte above each of those limits.  `pick_tile` restates the host's tile choice
(fg_abi.cu: pick_tile, init_device), so every builder knows the tile its batch gets, and the `*_rounds` functions restate
the round logic of the kernels, so a test can require the exact path every line takes.

All builders are seeded and return numpy (data uint8, offsets int32) batches, as oracle.pack does.
"""
from __future__ import annotations

import numpy as np

R5, LTSV, GELF, R3164 = 0, 1, 2, 3
LINES_PER_CTA = 64
LTSV_SLOTS = 64 * 24          # kLtsvStageSlots: one slot per TAB-separated part per round
GELF_SLOTS = 64 * 16          # kGelfStageSlots: one slot per top-level member per round
GELF_LOCAL_MEMBERS = 24       # kMaxLocalMembers: a line with more members goes to the exact parser
FIXED_MAX_TILE = 65024        # LTSV, GELF and RFC3164: tile positions are packed into 16 bits
TS = b"2015-08-05T15:53:45.637824Z"
R5_HEAD = b"<13>1 " + TS + b" h a p m "


# ---- the tile a call gets ------------------------------------------------------------------------------------------

def max_tile5(smem_optin: int) -> int:
    """RFC5424 tile limit from cudaDevAttrMaxSharedMemoryPerBlockOptin: the tile plus its 1/8 bitmap plus 1 KiB of static
    shared memory must fit (init_device).  227 KiB (H100) gives 180224."""
    t = min(smem_optin - 1024, 200 * 1024) & ~1023
    return ((t - 1024) * 8 // 9) & ~1023


H100_MAX_TILE5 = max_tile5(227 * 1024)


def pick_tile(fmt: int, total_bytes: int, n: int, max5: int = H100_MAX_TILE5) -> int:
    """The staging tile of a parse launch over n lines of total_bytes: mean * 64 * 1.02 + 512, rounded up to 512,
    clamped to [8192, format maximum]."""
    mean = total_bytes / n if n > 0 else 0.0
    gran = 8 * LINES_PER_CTA
    t = int(mean * LINES_PER_CTA * 1.02) + gran
    t = (t + gran - 1) // gran * gran
    return min(max(t, 8192), max5 if fmt == R5 else FIXED_MAX_TILE)


def batch_tile(fmt: int, offsets: np.ndarray) -> int:
    n = len(offsets) - 1
    return pick_tile(fmt, int(offsets[-1] - offsets[0]), n)


def pack(lines: list[bytes]) -> tuple[np.ndarray, np.ndarray]:
    offs = np.zeros(len(lines) + 1, dtype=np.int32)
    offs[1:] = np.cumsum([len(l) for l in lines])
    data = np.frombuffer(b"".join(lines) or b"\0", dtype=np.uint8).copy()[: int(offs[-1])]
    return data, offs


def lines_of(data: np.ndarray, offsets: np.ndarray) -> list[bytes]:
    return [bytes(data[offsets[i]:offsets[i + 1]]) for i in range(len(offsets) - 1)]


def _word(rng, n: int) -> bytes:
    return bytes(rng.integers(97, 123, n, dtype=np.uint8))


# ---- line makers of an exact length ----------------------------------------------------------------------------------

def r5_line(length: int, rng, tail: bool = False) -> bytes:
    """A regular RFC5424 line (the fast walker takes it) of exactly `length` bytes.  tail=False: one short SD pair and a
    long message; tail=True: a padding value first, then `k="v"` and the message at the far end of the line."""
    if tail:
        pre, post = R5_HEAD + b'[id a="', b'" k="v"] mm'
    else:
        pre, post = R5_HEAD + b'[id k="v"] ', b""
    pad = length - len(pre) - len(post)
    assert pad >= 1, length
    return pre + _word(rng, pad) + post


def ltsv_line(length: int, parts: int, rng) -> bytes:
    """A valid LTSV line with exactly `parts` TAB-separated parts and `length` bytes (time, host, then 4-byte `kX:v`
    parts; the message value takes the slack)."""
    head = [b"time:1438790025.5", b"host:h"] + [b"k%x:v" % (k % 16) for k in range(max(parts - 3, 0))]
    head = head[:parts - 1] if parts >= 1 else []
    pre = b"\t".join(head) + (b"\tmessage:" if head else b"message:")
    pad = length - len(pre)
    assert pad >= 1, (length, parts)
    return pre + _word(rng, pad)


def gelf_line(length: int, members: int, rng, long_numbers: int = 0) -> bytes:
    """A valid GELF line with exactly `members` top-level members and `length` bytes; `long_numbers` of the extra members
    are numbers of more than 6 bytes (the kernel lists those from the back of its number list), the others short ones."""
    assert members >= 3
    extra = []
    for k in range(members - 3):
        v = b"%d.25" % (1000000 + k) if k < long_numbers else b"%d" % (k % 100)
        extra.append(b'"_f%d":%s' % (k, v))
    pre = b'{"version":"1.1","host":"h",' + b"".join(e + b"," for e in extra) + b'"short_message":"'
    post = b'"}'
    pad = length - len(pre) - len(post)
    assert pad >= 1, (length, members)
    return pre + _word(rng, pad) + post


def r3164_line(length: int, rng) -> bytes:
    pre = b"<13>Aug  6 11:15:24 host app: "
    pad = length - len(pre)
    assert pad >= 1, length
    return pre + _word(rng, pad)


MAKERS = {R5: lambda L, rng: r5_line(L, rng), LTSV: lambda L, rng: ltsv_line(L, 3, rng),
          GELF: lambda L, rng: gelf_line(L, 4, rng), R3164: r3164_line}
SHORT = {R5: (60, 90), LTSV: (40, 70), GELF: (60, 90), R3164: (45, 80)}


# ---- batch assembly --------------------------------------------------------------------------------------------------

class Batch:
    """Lines appended CTA by CTA; `at` is the byte offset of the next line."""

    def __init__(self, fmt: int, seed: int):
        self.fmt = fmt
        self.rng = np.random.default_rng(seed)
        self.lines: list[bytes] = []
        self.at = 0

    def add(self, line: bytes) -> int:
        self.lines.append(line)
        self.at += len(line)
        return len(self.lines) - 1

    def short(self, extra: int = 0) -> int:
        lo, hi = SHORT[self.fmt]
        return self.add(MAKERS[self.fmt](int(self.rng.integers(lo, hi)) + extra, self.rng))

    def short_to_align(self, a: int) -> int:
        """a short line whose end leaves the next line at byte offset = a (mod 16)"""
        lo, _ = SHORT[self.fmt]
        L = lo + (a - (self.at + lo)) % 16
        return self.add(MAKERS[self.fmt](L, self.rng))

    def finish_cta(self) -> None:
        while len(self.lines) % LINES_PER_CTA:
            self.short()

    def fill_to_tile(self, tile: int) -> None:
        """Append whole CTAs of filler lines until pick_tile gives exactly `tile` for the batch."""
        self.finish_cta()
        lo, hi = SHORT[self.fmt]
        for _ in range(100_000):
            t = pick_tile(self.fmt, self.at, len(self.lines))
            if t == tile:
                return
            mean = self.at / len(self.lines)
            want = (tile - 768) / (LINES_PER_CTA * 1.02)
            L = int(self.rng.integers(lo, hi)) if mean > want else int(min(3 * want, tile // 2))
            self.add(MAKERS[self.fmt](L, self.rng))
        raise AssertionError(f"no filler reaches tile {tile}")

    def pack(self) -> tuple[np.ndarray, np.ndarray]:
        return pack(self.lines)


# ---- restated round logic: which path each line takes -----------------------------------------------------------------

def aligned_span(offsets: np.ndarray, i: int) -> int:
    return int(offsets[i + 1]) - (int(offsets[i]) & ~15)


def r5_tile_wide(offsets: np.ndarray, tile: int) -> set[int]:
    """parse5424_kernel: a line that does not fit the tile alone (r == 0) goes to the wide kernel.  Every line that is
    ever the first pending one of a round fits iff its own span from its aligned start fits, so this is exact."""
    return {i for i in range(len(offsets) - 1) if aligned_span(offsets, i) > tile}


def r5_long_wide(lines: list[bytes], strip_eol: bool = False) -> set[int]:
    """parse5424_kernel: a line of more than 65535 bytes (terminator stripped) goes to the wide kernel (u16 positions)."""
    def stripped(l: bytes) -> int:
        if strip_eol and l.endswith(b"\n"):
            l = l[:-1]
            if l.endswith(b"\r"):
                l = l[:-1]
        return len(l)
    return {i for i, l in enumerate(lines) if stripped(l) > 65535}


def r3164_tile_split(offsets: np.ndarray, tile: int) -> tuple[int, int]:
    """parse3164_kernel runs ONE round per CTA: the prefix of lines that fits the tile is read from it, the rest from
    global memory.  -> (lines from the tile, lines from global memory)."""
    n = len(offsets) - 1
    from_tile = 0
    for first in range(0, n, LINES_PER_CTA):
        last = min(n, first + LINES_PER_CTA)
        base = int(offsets[first]) & ~15
        r = 0
        while first + r < last and int(offsets[first + r + 1]) - base <= tile:
            r += 1
        from_tile += r
    return from_tile, n - from_tile


def slot_rounds(offsets: np.ndarray, tile: int, parts: list[int], cap: int, cut_to_direct: bool,
                direct_lines: set[int] = frozenset()) -> dict:
    """The round loop of parse_ltsv_kernel (cut_to_direct=True) and parse_gelf_kernel (False).  parts[i] = slots line i
    needs (LTSV: TAB-separated parts; GELF: members of a regular line, 0 for a line the exact parser takes).
    -> {"rounds": TMA rounds, "off_tile": lines taken by the direct / slow path for not fitting, "cuts": rounds cut by
    the slot cap, "direct_next": LTSV lines with more parts than slots}."""
    n = len(offsets) - 1
    st = {"rounds": 0, "off_tile": 0, "cuts": 0, "direct_next": 0, "in_round_direct": 0}
    for first in range(0, n, LINES_PER_CTA):
        last = min(n, first + LINES_PER_CTA)
        cur, direct_next = first, False
        while cur < last:
            base = int(offsets[cur]) & ~15
            r = 0
            if not direct_next:
                while cur + r < last and int(offsets[cur + r + 1]) - base <= tile:
                    r += 1
            if r == 0:
                direct_next = False
                st["off_tile"] += 1
                cur += 1
                continue
            st["rounds"] += 1
            run, r2 = 0, 0
            for k in range(r):
                if run + parts[cur + k] > cap:
                    break
                run += parts[cur + k]
                r2 += 1
            if r2 < r:
                st["cuts"] += 1
            if r2 == 0:
                assert cut_to_direct, "a GELF line holds at most kMaxLocalMembers < kGelfStageSlots members"
                direct_next = True
                st["direct_next"] += 1
                continue
            st["in_round_direct"] += sum(1 for k in range(r2) if cur + k in direct_lines)
            cur += r2
    return st


def stale_rounds(offsets: np.ndarray, tile: int) -> int:
    """Rounds (cut by bytes only) whose copy, rounded up to 16 bytes, is 16 mod 32 and shorter than an earlier round of
    the same CTA: the classifier's last granule then holds bytes an earlier round copied."""
    n, hits = len(offsets) - 1, 0
    for first in range(0, n, LINES_PER_CTA):
        last = min(n, first + LINES_PER_CTA)
        cur, longest = first, 0
        while cur < last:
            base = int(offsets[cur]) & ~15
            r = 0
            while cur + r < last and int(offsets[cur + r + 1]) - base <= tile:
                r += 1
            if r == 0:
                cur += 1
                continue
            nbytes = (int(offsets[cur + r]) - base + 15) & ~15
            hits += nbytes % 32 == 16 and nbytes + 16 <= longest
            longest = max(longest, nbytes)
            cur += r
    return hits


def ltsv_parts(lines: list[bytes]) -> list[int]:
    return [l.count(b"\t") + 1 for l in lines]


# ---- tile fit: every alignment, first line of a CTA and after a cut round, several rounds around r == 0 ----------------

def tile_fit(fmt: int, tile: int, seed: int) -> tuple[np.ndarray, np.ndarray, dict]:
    """Long lines whose span from their aligned start is tile - 1, tile and tile + 1, with the start at every offset
    mod 16: as the first line of a CTA, as the first line after a round that was cut before it, and CTAs of >= 3 TMA
    rounds with an r == 0 line between them.  Filler CTAs make pick_tile choose exactly `tile`."""
    B = Batch(fmt, seed)
    maker = MAKERS[fmt]
    targets = []

    def long_at(a: int, d: int) -> None:
        B.short_to_align(a)
        targets.append((B.add(maker(tile + d - a, B.rng)), d))

    for a in range(16):
        for d in (-1, 0, 1):
            # first line of a CTA: the last line of the previous CTA sets the alignment
            while len(B.lines) % LINES_PER_CTA != LINES_PER_CTA - 1:
                B.short()
            long_at(a, d)
            # after a round that was cut: 19 short lines, the aligning one, then the long one
            for _ in range(19):
                B.short()
            long_at(a, d)
            B.finish_cta()
    # >= 3 TMA rounds with r == 0 lines between them: short | fit | over | fit | short | over | fit | short
    for a in (0, 7, 15):
        for _ in range(4):
            B.short()
        for d in (0, 1, -1, 0, 1, 0):
            long_at((a + 5 * d) % 16, d)
            if d == 0:
                B.short()
        B.finish_cta()
    B.fill_to_tile(tile)
    data, offs = B.pack()
    assert batch_tile(fmt, offs) == tile
    over = [i for i, d in targets if d > 0]
    assert r5_tile_wide(offs, tile) == set(over)  # the same test decides r == 0 in every format
    return data, offs, {"tile": tile, "over": over, "fit": [i for i, d in targets if d <= 0]}


# ---- stale bytes in the odd granule of a tile ----------------------------------------------------------------------

DELIMS = {R5: b'"\\=] ', LTSV: b"\t:", GELF: b'"\\:, '}


def stale_granule(fmt: int, seed: int) -> tuple[np.ndarray, np.ndarray, int]:
    """CTAs of two rounds: round 1 fills the tile with lines full of the format's delimiters (plus ':' and TAB), round
    2 is short and its byte count, rounded up to 16, is 16 mod 32, so the classifier reads a granule the round did not
    copy — bytes round 1 left there.  Round 2 ends at every residue of 1..16 mod 32 from its base."""
    tile = 8192
    B = Batch(fmt, seed)
    rng = B.rng
    dl = DELIMS[fmt] + (b":" if fmt == GELF else b"\t:")  # a raw TAB would send a GELF line to the exact parser

    def noisy(L: int) -> bytes:
        if fmt == R5:  # one SD value with escaped delimiters, so the line stays valid
            body = b"".join(b"\\" + bytes([c]) if c in b'"\\]' else bytes([c]) for c in rng.choice(list(dl), L))
            pre = R5_HEAD + b'[id k="'
            return (pre + body)[: L - 4].rstrip(b"\\") + b'"] m'
        if fmt == LTSV:
            parts, n = [b"time:1438790025.5", b"host:h"], 0
            while sum(len(p) + 1 for p in parts) < L:
                parts.append(b"k%d:%s" % (n, bytes(rng.choice(list(b": ab"), 4).astype(np.uint8))))
                n += 1
            return b"\t".join(parts)[:L]
        body = b"".join(b"\\" + bytes([c]) if c in b'"\\' else bytes([c]) for c in rng.choice(list(dl), L))
        pre = b'{"version":"1.1","host":"h","short_message":"'
        return (pre + body)[: L - 2].rstrip(b"\\") + b'"}'

    for resid in range(1, 17):
        for variant in range(2):
            B.finish_cta()
            start = B.at
            # round 1: ~tile bytes of noisy lines (the last one does not fit with the rest)
            for _ in range(LINES_PER_CTA - 6):
                if B.at - (start & ~15) > tile - 400:
                    break
                B.add(noisy(int(rng.integers(100, 200))))
            # this line does not fit behind round 1: round 2 starts with it
            r2_base = B.at & ~15
            B.add(noisy(tile - (B.at - (start & ~15)) + 50 + variant * 30))
            # round 2: short lines; the CTA's last line ends at `resid` mod 32 from round 2's base
            while len(B.lines) % LINES_PER_CTA != LINES_PER_CTA - 1:
                B.short()
            L = SHORT[fmt][0] + (resid - (B.at + SHORT[fmt][0] - r2_base)) % 32
            B.add(MAKERS[fmt](L, rng))
    B.fill_to_tile(tile)
    data, offs = B.pack()
    return data, offs, tile


# ---- RFC5424: 16-bit positions ------------------------------------------------------------------------------------------

R5_TILE_16BIT = 66560  # holds a 65536-byte line plus its alignment and terminator


def r5_sixteen_bit(seed: int) -> tuple[list[bytes], int]:
    """Lines of 65534, 65535 and 65536 bytes, with the SD pair and the message at the far end (positions near 65535 are
    stored) and with a message of exactly 65535 bytes at the end, between short lines; the batch gets a tile that holds
    all of them, so only the 16-bit limit decides which lines go wide."""
    B = Batch(R5, seed)
    for a in (0, 5, 15):
        for L in (65534, 65535, 65536):
            B.short_to_align(a)
            B.add(r5_line(L, B.rng, tail=True))
            B.short()
    B.short()
    B.add(R5_HEAD + b"- " + _word(B.rng, 65535 - len(R5_HEAD) - 2))
    B.add(R5_HEAD + b"- " + _word(B.rng, 65535))  # the message alone is 65535 bytes
    B.finish_cta()
    B.fill_to_tile(R5_TILE_16BIT)
    return B.lines, R5_TILE_16BIT


def r5_max_tile(seed: int) -> list[bytes]:
    """Ten CTAs of 2.8-5.2 KB lines: the mean clamps pick_tile at the RFC5424 maximum of any device (the formula asks
    for ~260 KB), a CTA's span is larger than that maximum, so rounds are cut at the largest tile; one CTA also holds
    lines of 65535 and 65536 bytes, and only the latter go wide."""
    rng = np.random.default_rng(seed)
    lines = [r5_line(int(rng.integers(2800, 5200)), rng) for _ in range(10 * LINES_PER_CTA)]
    for k, L in zip(range(200, 264, 9), (65535, 65536) * 4):
        lines[k] = r5_line(L, rng, tail=True)
    return lines


def with_terminators(lines: list[bytes], crlf: bool) -> bytes:
    return b"".join(l + (b"\r\n" if crlf else b"\n") for l in lines)


# ---- LTSV: slots, the direct path, 16-bit spans ------------------------------------------------------------------------

def ltsv_slots(seed: int) -> tuple[np.ndarray, np.ndarray, dict]:
    """CTAs whose part totals are 1535, 1536 and 1537 (the last one is cut into two rounds); a first line with more
    parts than slots (the direct_next path, the TMA round is issued before the cut is known) followed by short lines, as
    the first line of a CTA and after a cut round; lines with a repeated `time` (the in-round direct path)."""
    B = Batch(LTSV, seed)
    rng = B.rng
    for total in (1535, 1536, 1537, 1535 + 64, 1536 + 64, 1537 + 64):
        B.finish_cta()
        per = [total // 64 + (1 if k < total % 64 else 0) for k in range(64)]
        rng.shuffle(per)
        for p in per:
            B.add(ltsv_line(p * 6 + 20, p, rng))
    for where in (0, 10, 63):
        B.finish_cta()
        for _ in range(where):
            B.short()
        B.add(ltsv_line(1537 * 5 + 60, 1537, rng))  # fits the tile, not the slots
        B.add(ltsv_line(1600 * 5 + 60, 1600, rng))
    B.finish_cta()
    for k in range(64):  # repeated `time`: the round-1 scanner inside a round
        B.add(b"time:1438790025.5\thost:h\ttime:1438790026.25\tmessage:m%d" % k if k % 9 == 4 else ltsv_line(60, 4, rng))
    B.fill_to_tile(16384)  # a CTA of 64 lines of ~24 parts fits the tile: the slots cut the round, not the bytes
    data, offs = B.pack()
    return data, offs, {"tile": 16384}


def ltsv_sixteen_bit(seed: int) -> tuple[np.ndarray, np.ndarray, int]:
    """Lines whose span from the aligned start is 65023, 65024 and 65025 under the 65024 tile (the last goes direct),
    and a value of exactly 65535 bytes."""
    B = Batch(LTSV, seed)
    for a in (0, 9):
        for d in (-1, 0, 1):
            while len(B.lines) % LINES_PER_CTA != LINES_PER_CTA - 1:
                B.short()
            B.short_to_align(a)  # the long line opens the next CTA at offset a (mod 16)
            B.add(ltsv_line(FIXED_MAX_TILE + d - a, 5, B.rng))
            B.short()
    B.add(b"time:1438790025.5\thost:h\tbig:" + _word(B.rng, 65535) + b"\tmessage:m")
    B.add(b"time:1438790025.5\thost:h\tmessage:" + _word(B.rng, 65535))
    B.fill_to_tile(FIXED_MAX_TILE)
    data, offs = B.pack()
    return data, offs, FIXED_MAX_TILE


# ---- LTSV schema placement -----------------------------------------------------------------------------------------------

LTSV_TYPES = ("bool", "f64", "i64", "u64")
TYPED_VALUE = {"bool": b"true", "f64": b"-0.5e3", "i64": b"-42", "u64": b"18446744073709551615", "string": b"s"}


def ltsv_schemas() -> list[tuple[str, dict, dict]]:
    """(label, schema, suffixes) on both sides of each staging limit: 64 / 65 keys, a name blob of 1024 / 1025 bytes, a
    suffix blob of 64 / 65 bytes.  The keys collide with the length and first-byte filters: many keys of one length and
    one first byte, names of 31 bytes and more (one length-filter bit), and the empty key."""
    def keys(n: int, blob: int) -> dict:
        out = {"": "u64"}
        k = 0
        while len(out) < n - 1:
            out["k%02d" % k] = LTSV_TYPES[k % 4]
            k += 1
        used = sum(len(x) for x in out)
        # the last key takes the rest of the blob: 31+ bytes, same first byte as the short keys
        out["k" + "L" * (blob - used - 1)] = "f64"
        return out

    base = keys(60, 600)
    suffix = {"bool": "_b", "f64": "_f", "i64": "_i", "u64": "_u"}
    s64 = {"bool": "_" + "b" * 15, "f64": "_" + "f" * 15, "i64": "_" + "i" * 15, "u64": "_" + "u" * 15}
    s65 = dict(s64, u64="_" + "u" * 16)
    return [("keys64", keys(64, 600), suffix), ("keys65", keys(65, 600), suffix),
            ("blob1024", keys(40, 1024), suffix), ("blob1025", keys(40, 1025), suffix),
            ("suffix64", base, s64), ("suffix65", base, s65)]


def ltsv_schema_lines(schema: dict, suffixes: dict, seed: int) -> list[bytes]:
    """Lines whose keys hit every schema key, suffixed keys of all four types, near misses of the filters (same length,
    same first byte, a 31+-byte name one byte off), typed values that parse and that do not."""
    rng = np.random.default_rng(seed)
    names = list(schema)
    out = []
    for k in range(600):
        parts = [b"time:1438790025.5", b"host:h"]
        for j in range(int(rng.integers(3, 9))):
            nm = names[int(rng.integers(0, len(names)))]
            ty = schema[nm]
            kind = int(rng.integers(0, 6))
            if kind == 0:  # the same length and first byte, not a key
                nm = (nm[:-1] + "Z") if nm else "Z"
            elif kind == 1:
                t = LTSV_TYPES[int(rng.integers(0, 4))]
                nm, ty = "x%d%s" % (j, suffixes[t]), t
            v = TYPED_VALUE[ty] if (kind != 2 or ty == "string") else b"notanumber"
            parts.append(nm.encode() + b":" + v)
        parts.append(b"message:m%d" % k)
        out.append(b"\t".join(parts))
    return out


# ---- GELF: slots, members per line, the two ends of the number list ---------------------------------------------------

def gelf_slots(seed: int) -> tuple[np.ndarray, np.ndarray, dict]:
    """CTAs whose member totals are 1023, 1024 and 1025 (the last one is cut); lines of 23, 24 and 25 members (25 goes
    to the exact parser); a round of 1024 members of which 832 are numbers, 704 of them longer than 6 bytes (the
    long-number end of the list passes the middle); and a round of 1024 members that are ALL numbers, so the
    short-number and long-number ends of the number list meet (nshort + nlong = kGelfStageSlots).  The all-number lines
    have no `host`, so they are decoded as errors, after their numbers went through the list."""
    B = Batch(GELF, seed)
    rng = B.rng
    for total in (1023, 1024, 1025):
        B.finish_cta()
        per = [total // 64 + (1 if k < total % 64 else 0) for k in range(64)]
        rng.shuffle(per)
        for p in per:
            B.add(gelf_line(p * 20 + 80, p, rng, long_numbers=int(rng.integers(0, p - 2))))
    for m in (23, 24, 25):
        B.finish_cta()
        for k in range(64):
            mm = m if k % 5 == 0 else 6
            B.add(gelf_line(mm * 22 + 80, mm, rng, long_numbers=(k * 7) % (mm - 2)))
    B.finish_cta()
    for k in range(64):  # 16 members each, 13 numbers: 11 long, 2 short
        B.add(gelf_line(16 * 20 + 80, 16, rng, long_numbers=11))
    B.finish_cta()
    for k in range(64):  # 16 members each, all numbers: 5 to 11 long, the rest short
        n_long = 5 + k % 7
        B.add(b"{" + b",".join(b'"_n%d":%s' % (j, b"%d.5" % (1000000 + j) if j < n_long else b"%d" % j)
                               for j in range(16)) + b"}")
    B.fill_to_tile(32768)  # a CTA of 64 lines of 16 members fits the tile: the slots cut the round, not the bytes
    data, offs = B.pack()
    return data, offs, {"tile": 32768}


def gelf_members(lines: list[bytes]) -> list[int]:
    """top-level members of the builders' lines (no nested objects, no ',' or ':' inside strings)"""
    return [l.count(b",") + 1 for l in lines]


# ---- lock-step mixes: one odd line at every lane position ------------------------------------------------------------

def lane_mix(fmt: int, seed: int) -> tuple[np.ndarray, np.ndarray]:
    """Warps of uniform lines with one odd line at lane 0..31 of the warp (both warps of a 64-line CTA)."""
    rng = np.random.default_rng(seed)
    if fmt == R3164:
        plain = lambda: r3164_line(int(rng.integers(50, 70)), rng)
        odd = [b"testhostname: 2020 Aug  6 11:15:24 UTC: appname 69 42 some test message",      # custom form
               b"<13>Aug  6 11:15:24 host app:  two  spaces   re-joined ",                       # re-join
               b"<13>2020 Aug 6 05:15:24 America/Sao_Paulo host app: zone",                      # zone
               b"<13>Aug  6 11:15:24 host app: " + _word(rng, 9000)]                               # from global memory
    elif fmt == LTSV:
        plain = lambda: ltsv_line(int(rng.integers(50, 70)), 4, rng)
        odd = [b"time:1438790025.5\thost:h\ttime:1438790026.25\tmessage:twice",
               ltsv_line(1537 * 5 + 60, 1537, rng)]
    else:
        plain = lambda: gelf_line(int(rng.integers(90, 110)), 5, rng, long_numbers=1)
        odd = [gelf_line(700, 25, rng, long_numbers=3),
               b'{"version":"1.1","host":"h","short_message":"raw\x01ctrl"}',
               b'{"version":"1.1", "host": "h" ,"short_message":"spaces","_n":1e400}']
    lines = []
    for o in odd:
        for lane in range(32):
            for w in range(2):
                for k in range(32):
                    lines.append(o if k == lane and (w == 0 or lane % 2 == 0) else plain())
    return pack(lines)


# ---- the fused GELF encoder --------------------------------------------------------------------------------------------

def enc_line(pairs: list[tuple[bytes, bytes]], rng, host: bytes = b"h", msg: bytes = b"m", elems: int = 1) -> bytes:
    if not pairs:
        return b"<13>1 " + TS + b" " + host + b" a p m - " + msg
    chunks = np.array_split(np.arange(len(pairs)), min(elems, len(pairs)))
    sd = b"".join(b"[e%d " % j + b" ".join(pairs[k][0] + b'="' + pairs[k][1] + b'"' for k in ch) + b"]"
                  for j, ch in enumerate(chunks))
    return b"<13>1 " + TS + b" " + host + b" a p m " + sd + b" " + msg


def enc_pair_counts(seed: int) -> list[bytes]:
    """0..40 pairs per line, so the segment count of a record crosses 56 and 112 at every kind of segment (pair names,
    values, escaped values, empty values that push no segment, the "unknown" literal of an empty host); one and three
    SD elements."""
    rng = np.random.default_rng(seed)
    out = []
    for n in range(41):
        for variant in range(6):
            pairs = []
            for k in range(n):
                v = [b"v", b"", b'q\\"x', _word(rng, int(rng.integers(1, 9)))][(k + variant) % 4]
                pairs.append((b"n%02d" % k, v))
            if variant % 2:
                rng.shuffle(pairs)
            host = b"-" if variant == 3 else (b"" if variant == 5 else b"host%d" % variant)
            line = enc_line(pairs, rng, host=host if host else b"h", msg=b"msg %d" % n, elems=1 + 2 * (variant % 2))
            if variant == 5:
                line = line.replace(b" h a p m", b"  a p m", 1)  # empty host field
            out.append(line)
    return out


def enc_duplicates(seed: int) -> list[bytes]:
    """23, 24 and 25 pairs (24 = kLocalPairs: more switch the encoder to its O(n^2) selection) with a duplicated name
    inside the first 24, across the boundary and after it; the last duplicate must win in both modes."""
    rng = np.random.default_rng(seed)
    out = []
    for n in (23, 24, 25, 26, 40):
        for first, second in ((0, 5), (3, 23), (10, 24), (23, 24), (24, 25), (0, n - 1), (n - 2, n - 1)):
            if second >= n:
                continue
            names = [b"d%02d" % k for k in range(n)]
            names[second] = names[first]
            for order in range(2):
                pairs = [(nm, b"val%d" % k) for k, nm in enumerate(names)]
                if order:
                    pairs = pairs[::-1]
                out.append(enc_line(pairs, rng, elems=1 + order))
        # three copies of one name spread over the whole line
        names = [b"t%02d" % k for k in range(n)]
        for k in (0, n // 2, n - 1):
            names[k] = b"same"
        out.append(enc_line([(nm, b"w%d" % k) for k, nm in enumerate(names)], rng, elems=2))
    return out


ENC_EXTRAS = [{"0": "zero"}, {"A": "upper"}, {"^": "caret"}, {"_": "under"}, {"_n01": "collides with _n01"},
              {"é": "e-acute"}, {"": "empty key"},
              {"0": "z", "A": "a", "^": "c", "_": "u", "_d03": "x", "é": "e", "": "", "zz": "last"}]


def enc_long_and_spans(seed: int) -> tuple[list[bytes], list[bytes]]:
    """(lines of >= 1008 bytes — length class 63 — around a few hundred short ones;
    a 256-line encoder span larger than the encoder tile min(4 * parse tile, RFC5424 maximum) inside a batch whose mean
    keeps the parse tile at 8192)."""
    rng = np.random.default_rng(seed)
    long_lines = []
    for k in range(300):
        L = 1000 + (k % 40) if k % 3 == 0 else int(rng.integers(60, 200))
        long_lines.append(r5_line(L, rng) if k % 2 else enc_line([(b"p%d" % j, _word(rng, 40)) for j in range(L // 50)], rng))
    span = [r5_line(70, rng) for _ in range(256 * 20)]
    for k in range(256 * 4, 256 * 5):  # one 256-line span of ~140 KB > 4 * 8192
        span[k] = r5_line(int(rng.integers(400, 700)), rng)
    return long_lines, span


def enc_lane_mix(seed: int) -> list[bytes]:
    """Warps of ordinary lines with one rejected line and one line of more than 24 pairs at lane 0..31."""
    rng = np.random.default_rng(seed)
    many = enc_line([(b"m%02d" % ((k * 7) % 30), b"v%d" % k) for k in range(30)], rng)
    bad = b"<13>1 " + TS + b" h a p m [broken"
    out = []
    for lane in range(32):
        warp = [enc_line([(b"a", b"1"), (b"b", b"2")], rng) for _ in range(32)]
        warp[lane] = many
        warp[(lane + 11) % 32] = bad
        out += warp
    return out


# ---- UTF-8 and framing seams of the device splitter --------------------------------------------------------------------

LEADS = [0xC2, 0xDF, 0xE0, 0xE1, 0xEC, 0xED, 0xEE, 0xEF, 0xF0, 0xF1, 0xF3, 0xF4]
SECONDS = [0x7F, 0x80, 0x8F, 0x90, 0x9F, 0xA0, 0xBF, 0xC0]
SEG = 8192


def utf8_probes() -> list[bytes]:
    """Every lead class with second bytes at the class bounds, complete and truncated by 1 to 3 bytes, and valid
    sequences followed by 1 to 4 stray continuation bytes."""
    out = []
    for lead in LEADS:
        need = 1 if lead < 0xE0 else (2 if lead < 0xF0 else 3)
        for b1 in SECONDS:
            full = bytes([lead, b1]) + b"\x80" * (need - 1)
            for cut in range(0, need + 1):
                out.append(full[: len(full) - cut])
    for seq in ("é", "日", "\U0001F680"):
        for deep in range(1, 5):
            out.append(seq.encode() + b"\x80" * deep)
    return out


def utf8_stream(delim: bytes, seed: int) -> bytes:
    """RFC5424 records holding one probe each, the probe starting at every offset mod 16; then probes that start 1..4
    bytes before an 8 KiB segment seam; delimiters as the first and last byte of a segment and of a 16-byte window;
    '\\r' + delimiter split across a seam.  Well below the 64 MiB chunk size."""
    rng = np.random.default_rng(seed)
    probes = utf8_probes()
    head = b"<13>1 " + TS + b" h a p m - "
    out = bytearray()

    def rec(body: bytes, cr: bool = False) -> None:
        out.extend(head + body + (b"\r" if cr else b"") + delim)

    for k, p in enumerate(probes):
        for off in range(16):
            # the probe starts at stream offset = off (mod 16)
            pad = (off - (len(out) + len(head))) % 16
            rec(b"x" * pad + p + b" tail" * (k % 2), cr=(k + off) % 5 == 0)
    for k, p in enumerate(probes):
        # the probe straddles (or ends right at) the next segment seam
        back = 1 + k % 4
        seam = (len(out) // SEG + 1) * SEG
        pad = seam - back - len(out) - len(head)
        if pad < 0:
            seam += SEG
            pad += SEG
        rec(b"y" * pad + p + b"z")
    for where in (0, -1, 15, 16, -16, -17):  # a delimiter at the first / last byte of a segment and of a window
        seam = (len(out) // SEG + 1) * SEG
        pad = seam + where - len(out) - len(head)
        if pad < 0:
            pad += SEG
        rec(b"w" * pad)
    for split in (0, 1):  # '\r' then the delimiter, the seam between them or before the '\r'
        seam = (len(out) // SEG + 1) * SEG
        pad = seam - 1 + split - len(out) - len(head)
        rec(b"v" * pad, cr=True)
    rec(_word(rng, 50))
    return bytes(out)
