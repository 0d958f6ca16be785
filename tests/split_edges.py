"""Streams for the front end every raw-stream call shares (fg_split_decode, fg_split_decode_framed and the four
fg_split_decode_encode_* calls): `split_stream` in fg_abi.cu and the kernels of fg_split.cu.  That front end frames the
stream at '\\n' or NUL, checks each record as core::str::from_utf8 does, and pipelines both over 64 MiB chunks.

Each builder gives the stream and where its probes sit; what the stream should frame into comes from the references:
record starts as oracle/pysplit.py frames them, and per-record validity as Python's strict `bytes.decode("utf-8")`
gives it.  Python's strict decoder and Rust's from_utf8 accept the same set (Unicode Table 3-7: no overlongs, no
surrogates, nothing above U+10FFFF).  `fast_expect` restates both with numpy for the exhaustive streams, whose ~12 M
records are too many for a per-record loop; the CPU tests hold it equal to pysplit.  Pure Python and numpy."""
from __future__ import annotations

import functools

import numpy as np

CHUNK = 64 << 20  # split_stream's pipeline chunk
LAG = 16          # the validated window lags this far behind the uploaded bytes (v1 = c1 - 16)
TS = b"2015-08-05T15:53:45.637824Z"
HEAD = b"<13>1 " + TS + b" h a p m - "  # an RFC5424 header without structured data: the rest of a record is its msg
INVALID_UTF8 = 76  # FG_ES_INVALID_UTF8
UTF8_ERROR_DUMP = b"E:Invalid UTF-8 input;out=0"
DELIMS = {"line": b"\n", "nul": b"\0"}

# ---- the references ------------------------------------------------------------------------------------------------


def expect(stream: bytes, delim: bytes):
    """pysplit's framing of `stream`: (record starts int32[n + 1], stripped records, utf8-valid flags)"""
    import pysplit
    return (pysplit.split_nul if delim == b"\0" else pysplit.split_lines)(stream)


def record_starts(stream: bytes | np.ndarray, delim: bytes) -> np.ndarray:
    """pysplit's record starts from numpy: 0, every byte after a delimiter, and the end of an unterminated stream"""
    a = np.frombuffer(stream, np.uint8) if isinstance(stream, (bytes, bytearray)) else stream
    if len(a) == 0:
        return np.zeros(1, np.int32)
    st = np.flatnonzero(a == delim[0]) + 1
    tail = [len(a)] if a[-1] != delim[0] else []
    return np.concatenate([[0], st, tail]).astype(np.int32)


def fast_expect(stream: bytes, delim: bytes) -> tuple[np.ndarray, np.ndarray]:
    """(record starts, utf8-valid flags) as `expect` gives them, without a per-record loop.  The whole stream is decoded
    once with errors="surrogateescape": every byte the strict decoder refuses becomes one of U+DC80..U+DCFF, which no
    valid text decodes to, and the delimiter is ASCII, so it decodes to itself and is never part of a refused sequence.
    A record is valid exactly when none of those code points lies between its delimiters."""
    starts = record_starts(stream, delim)
    n = len(starts) - 1
    u = np.frombuffer(stream.decode("utf-8", "surrogateescape").encode("utf-32-le", "surrogatepass"), np.uint32)
    is_delim = u == delim[0]
    bad = np.flatnonzero((u >= 0xDC80) & (u <= 0xDCFF))
    rec = np.cumsum(is_delim)[bad] - is_delim[bad]  # the record of each refused byte: the delimiters before it
    return starts, np.bincount(rec, minlength=n)[:n] == 0


# ---- every short sequence, each in a record of its own ----------------------------------------------------------------

FOUR_B3 = (0x41, 0x7F, 0x80, 0x8F, 0x90, 0xBF, 0xC0)  # the class bounds of a fourth byte
FOUR_B2 = (0x7F, 0x80, 0xBF, 0xC0)                    # ... and of a third
EXHAUSTIVE_BATCH = 1 << 21                            # candidates per stream (one device call each)


def _grid(*axes) -> np.ndarray:
    """every combination of the byte axes, the last axis fastest: uint8[n, len(axes)]"""
    g = np.meshgrid(*[np.asarray(a, np.uint8) for a in axes], indexing="ij")
    return np.stack([x.ravel() for x in g], axis=1)


@functools.lru_cache(maxsize=2)
def exhaustive_candidates(delim: bytes) -> tuple[np.ndarray, np.ndarray]:
    """(bytes uint8[n, 4], lengths int[n]) of every candidate, in this order:
    - every b0 b1 b2 with b0 in 0x80..0xFF (8.3 M);
    - every F0..F4 b1 b2 b3 with b1, b2 over all bytes and b3 at the bounds FOUR_B3;
    - every F0..F4 b1 b2 b3 with b1, b3 over all bytes and b2 at the bounds FOUR_B2;
    - every b0 and b0 b1 with b0 in 0x80..0xFF: C0 and C1 followed by every byte, F5..FF leads, truncated sequences.
    "Every byte" leaves out the delimiter, so that each candidate is one record."""
    anyb = [b for b in range(256) if b != delim[0]]
    high = range(0x80, 0x100)
    four = range(0xF0, 0xF5)
    parts = [_grid(high, anyb, anyb), _grid(four, anyb, anyb, FOUR_B3), _grid(four, anyb, FOUR_B2, anyb),
             _grid(high), _grid(high, anyb)]
    n = sum(len(p) for p in parts)
    cand = np.zeros((n, 4), np.uint8)
    clen = np.zeros(n, np.int64)
    at = 0
    for p in parts:
        cand[at:at + len(p), :p.shape[1]] = p
        clen[at:at + len(p)] = p.shape[1]
        at += len(p)
    return cand, clen


EXHAUSTIVE_COUNT = 128 * 255 * 255 + 5 * 255 * 255 * len(FOUR_B3) + 5 * 255 * len(FOUR_B2) * 255 + 128 + 128 * 255
EXHAUSTIVE_BATCHES = -(-EXHAUSTIVE_COUNT // EXHAUSTIVE_BATCH)


def utf8_exhaustive_batch(delim: bytes, k: int) -> tuple[bytes, np.ndarray, np.ndarray]:
    """Candidates [k * EXHAUSTIVE_BATCH, (k + 1) * EXHAUSTIVE_BATCH) of exhaustive_candidates, one record each:
    ASCII padding, the candidate, one ASCII byte after it in every 5th record, '\\r' before the delimiter in every 7th
    record under line framing.  Candidate r (counted over all batches) starts at an offset = r (mod 16).
    Returns (stream, candidate offsets, candidate lengths)."""
    cand, clen = exhaustive_candidates(delim)
    r = np.arange(k * EXHAUSTIVE_BATCH, min((k + 1) * EXHAUSTIVE_BATCH, len(clen)))
    cand, clen = cand[r], clen[r]
    suffix = (r % 5 == 0).astype(np.int64)
    cr = (r % 7 == 0).astype(np.int64) if delim == b"\n" else np.zeros(len(r), np.int64)
    body = clen + suffix + cr + 1  # from the candidate to the delimiter, inclusive
    # the candidate of record r starts at c_r = r (mod 16); record r + 1 starts at c_r + body_r, so its padding
    # (1 - body_r) mod 16 brings c_{r+1} to r + 1 (mod 16)
    pad = np.empty(len(r), np.int64)
    pad[0] = r[0] % 16
    pad[1:] = (1 - body[:-1]) % 16
    ends = np.cumsum(pad + body)
    at = ends - body  # candidate offsets
    out = np.full(int(ends[-1]), ord("x"), np.uint8)
    for j in range(4):
        m = clen > j
        out[at[m] + j] = cand[m, j]
    out[(at + clen)[suffix == 1]] = ord("a")
    out[(ends - 2)[cr == 1]] = ord("\r")
    out[ends - 1] = delim[0]
    return out.tobytes(), at, clen


def utf8_exhaustive(delim: bytes):
    """utf8_exhaustive_batch for every batch in turn"""
    for k in range(EXHAUSTIVE_BATCHES):
        yield utf8_exhaustive_batch(delim, k)


# ---- sequences against their neighbours ---------------------------------------------------------------------------------


def utf8_in_context(delim: bytes) -> tuple[bytes, list[tuple[str, int]]]:
    """Probes next to delimiters and to each other, each with its first byte at every offset mod 16:
    - a valid character followed by 1-4 stray continuation bytes;
    - a continuation byte as the first byte after a delimiter (the record before ending in a character, a lead, '\\r');
    - a lead byte, or a sequence one byte short, as the last byte before the delimiter and before "\\r\\n";
    - two invalid sequences in one record;
    - an invalid sequence in each of two adjacent records, and invalid / valid / invalid records, inside one 16-byte
      window.
    Returns (stream, [(probe name, offset of its first byte)])."""
    out = bytearray()
    probes = []
    line = delim == b"\n"

    def rec(body: bytes, cr: bool = False) -> None:
        out.extend(body + (b"\r" if cr and line else b"") + delim)

    def aligned(off: int, name: str, head: bytes = HEAD) -> bytes:
        """head + padding such that the next byte sits at `off` (mod 16)"""
        pad = (off - len(out) - len(head)) % 16
        probes.append((name, len(out) + len(head) + pad))
        return head + b"x" * pad

    for off in range(16):
        for ch in ("é", "日", "\U0001F680"):
            for k in range(1, 5):
                rec(aligned(off, f"stray{k}") + ch.encode() + b"\x80" * k + b" tail")
        for before in ("日".encode(), b"\xe6", b"\xf0\x9f\x9a", b"ok"):
            cr = line and before == b"ok"
            pad = (off - len(out) - len(HEAD) - len(before) - cr - 1) % 16  # the next record starts at `off`
            rec(HEAD + b"x" * pad + before, cr=cr)
            probes.append(("first", len(out)))
            rec(b"\x80" + b"\xbf" * (off % 3) + b" rest")
        for last in (b"\xc3", b"\xe6", b"\xf0", b"\xe6\x97", b"\xf0\x9f\x9a"):
            for cr in (False, True):
                rec(aligned(off, "last") + last, cr=cr)
        rec(aligned(off, "two") + b"\xff ok \xc3(" + b" and \xed\xa0\x80 end")
        rec(aligned(off, "two") + b"\xe0\x9f\xbf" + "é".encode() + b"\xf4\x90\x80\x80")
        # adjacent short records inside one 16-byte window
        rec(aligned(off, "window", b"") + b"\xff")
        rec(b"\xc0\xaf")
        rec(aligned(off, "window", b"") + b"a\xfe")
        rec("é".encode())
        rec(b"\xed\xa0\x80")
        rec(b"ok")
        rec(aligned(off, "window", b"") + "日".encode())
        rec(b"\x80")
        rec("é".encode())
    rec(HEAD + b"end")
    return bytes(out), probes


# ---- the 64 MiB chunk seam ----------------------------------------------------------------------------------------------

SEAM_EVENTS = {
    "delim": None,           # the delimiter itself
    "cr_delim": b"\r",       # '\r' + the delimiter
    "stray": b"\x80",        # a continuation byte no lead claims
    "lead": b"\xf0",         # a lone 4-byte lead (reads 3 bytes ahead)
    "char2": "é".encode(),
    "char3": "日".encode(),
    "char4": "\U0001F680".encode(),
    "overlong": b"\xe0\x80\x80",
    "surrogate": b"\xed\xa0\x80",
}
SEAM_WHERE = range(-20, 20)
SEAM_QUIET = 4096  # no delimiter of the base stream within this distance of the seam


def seam_event(delim: bytes, kind: str) -> bytes:
    e = SEAM_EVENTS[kind]
    return delim if e is None else (e + delim if kind == "cr_delim" else e)


def records_layout(total: int, rng, lo: int, hi: int, quiet: list[tuple[int, int]] = ()) -> np.ndarray:
    """record ends (exclusive) of records of lengths drawn in [lo, hi) that fill `total` bytes, with no record end
    inside a `quiet` range (there the record before is longer) and the last record at least `lo` long"""
    lens = rng.integers(lo, hi, total // lo + 2)
    ends = np.cumsum(lens)
    ends = ends[ends <= total - lo]
    for a, b in quiet:
        ends = ends[(ends <= a) | (ends > b)]
    return np.append(ends, total)


def fill_records(out: np.ndarray, ends: np.ndarray, delim: bytes, rng, terminated: bool = True) -> np.ndarray:
    """`out` (uint8) filled with RFC5424 records with lowercase messages that end at `ends` (the last end = len(out)); the
    last record without its delimiter unless `terminated`"""
    total = len(out)
    out[:] = rng.integers(ord("a"), ord("z") + 1, total, dtype=np.uint8)
    starts = np.concatenate([[0], ends[:-1]])
    h = np.frombuffer(HEAD, np.uint8)
    out[starts[:, None] + np.arange(len(h))] = h
    out[ends[:-1] - 1] = delim[0]
    if terminated:
        out[total - 1] = delim[0]
    return out


@functools.lru_cache(maxsize=2)
def seam_base(delim: bytes) -> np.ndarray:
    total = CHUNK + (64 << 10)
    rng = np.random.default_rng(11)
    ends = records_layout(total, rng, 1000, 8000, [(CHUNK - SEAM_QUIET, CHUNK + SEAM_QUIET)])
    out = fill_records(np.empty(total, np.uint8), ends, delim, rng)
    out.flags.writeable = False
    return out


def chunk_seam(delim: bytes, where: int, kind: str) -> tuple[np.ndarray, int]:
    """64 MiB + 64 KiB of RFC5424 records of 1-8 KB with lowercase messages, one of which spans the first chunk
    seam; the event `kind` overwrites its message at offset CHUNK + where.  Returns (stream, event offset)."""
    out = seam_base(delim).copy()
    e = np.frombuffer(seam_event(delim, kind), np.uint8)
    out[CHUNK + where:CHUNK + where + len(e)] = e
    return out, CHUNK + where


# ---- records longer than a chunk, and stream lengths around the chunk multiples -----------------------------------------

LEN_DELTAS = (-1, 0, 1, 15, 16, 17)


def _one_long(delim: bytes, length: int, marks: dict[int, bytes], seed: int) -> np.ndarray:
    """a 300-byte record, a record of `length` bytes (its delimiter included) starting at 300, and a 300-byte record;
    `marks` overwrite the long record's message at absolute offsets"""
    total = 300 + length + 300
    out = fill_records(np.empty(total, np.uint8), np.array([300, 300 + length, total]), delim, np.random.default_rng(seed))
    for at, b in marks.items():
        out[at:at + len(b)] = np.frombuffer(b, np.uint8)
    return out


def long_records(delim: bytes):
    """(label, stream) pairs:
    - one record of 64 MiB + 100 bytes;
    - one of 130 MiB, which spans three chunks: the middle chunk holds no delimiter; also with valid 2-, 3- and 4-byte
      characters across both seams and in the middle chunk, and with one invalid byte in the middle chunk;
    - streams of k * 64 MiB + d bytes (k = 1, 2; d in LEN_DELTAS) of 1-8 KB records, ending with and without the
      delimiter; k = 1, d = 1 with the delimiter is a last chunk that is the delimiter alone."""
    yield "64M+100", _one_long(delim, CHUNK + 100, {}, 1)
    big = 130 << 20
    yield "130M", _one_long(delim, big, {}, 2)
    yield "130M-utf8", _one_long(delim, big, {CHUNK - 2: "日".encode(), CHUNK + (32 << 20): "\U0001F680".encode(),
                                              2 * CHUNK - 1: "é".encode(), 2 * CHUNK + 7: "\U0001F680".encode()}, 3)
    yield "130M-invalid", _one_long(delim, big, {CHUNK - 2: "日".encode(), CHUNK + (32 << 20): b"\xff"}, 4)
    for k in (1, 2):
        for d in LEN_DELTAS:
            total = k * CHUNK + d
            rng = np.random.default_rng(100 + 10 * k + d)
            ends = records_layout(total, rng, 1000, 8000)
            for term in (True, False):
                yield f"{k}x64M{d:+d}-{'term' if term else 'open'}", fill_records(np.empty(total, np.uint8), ends, delim, rng, term)


# ---- record counts around max_batch_lines -------------------------------------------------------------------------------


def capacity_streams(max_lines: int, delim: bytes):
    """(label, stream, records) triples: max_lines - 1, max_lines and max_lines + 1 short records, each terminated and
    unterminated; and max_lines records of at least 20 KB (and long enough for the stream to pass one chunk), terminated,
    whose last delimiter falls in the second chunk."""
    for n in (max_lines - 1, max_lines, max_lines + 1):
        body = b"".join(HEAD + b"m%d" % i + delim for i in range(n))
        yield f"{n}-term", body, n
        yield f"{n}-open", body[:-1], n
    rng = np.random.default_rng(5)
    lo = max(20_000, CHUNK // max_lines * 5 // 4)
    lens = rng.integers(lo, lo + 1000, max_lines)
    ends = np.cumsum(lens)
    yield f"{max_lines}-long-term", fill_records(np.empty(int(ends[-1]), np.uint8), ends, delim, rng).tobytes(), max_lines
