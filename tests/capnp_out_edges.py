"""Lines for the edges of the fused Cap'n Proto encoder (test infrastructure, pure Python, no GPU): a model of the segment
list build_capnp (fg_capnp_encode.cu) makes of a record, and lines whose records place every kind of entry on the window
boundaries of that list (kMaxCapSegs = 64 entries per window, a longer record is rebuilt window by window) or lay their
objects out over several message segments on purpose."""
from __future__ import annotations

import struct

import capnp_oracle as O

R5, LTSV, GELF, R3 = 0, 1, 2, 3
WINDOW = 64
# 0-based entry indices around the window boundaries: the last entry of the first and second window and the first entry
# of the second and third
BOUNDARIES = (WINDOW - 1, WINDOW, 2 * WINDOW - 1, 2 * WINDOW)
TOTALS = (63, 64, 65, 127, 128, 129, 191, 192, 193)
TYPED = {"counter": "u64", "score": "i64", "mean": "f64", "done": "bool"}
SUFFIXES = {"u64": "_u64", "i64": "_i64", "f64": "_f64", "bool": "_bool"}
TS = b"2015-08-05T15:53:45.637824Z"
EXTRA = {"_x": "a\tb:c", "y": "1", "z": ""}  # keys as given, an empty value

# the kinds of entry each source can put on a window boundary: a pair list's tag and words, a landing pad, the texts of
# its pairs and of output.capnp_extra (RFC3164 records have no pairs and never reach one)
_PAIRED = {"tag", "pw0", "pw1", "kptr", "vptr", "pad", "us", "end", "body:key", "body:value", "body:xkey", "body:xvalue"}
KINDS = {R5: _PAIRED, LTSV: _PAIRED | {"suffix"}, GELF: _PAIRED | {"json"}, R3: set()}
# (window start, message segment of the list) of an entry right after a whole pair list's words.  An RFC5424 record
# cannot drop an entry before its pair list (every field is a text), an LTSV record only two: the window lines do not
# reach 64 after a list in segment 1 for RFC5424, nor 128 for LTSV.
AFTER_LIST = {R5: {(64, 0), (128, 0), (128, 1)}, LTSV: {(64, 0), (128, 0), (64, 1)},
              GELF: {(64, 0), (128, 0), (64, 1), (128, 1)}, R3: set()}


def _json(text: bytes) -> bool:
    """a GELF string whose text holds a byte JSON must escape came from a span with escapes"""
    return any(c < 0x20 or c in b'"\\' for c in text)


def _key(src: int, key: bytes) -> tuple[bytes, bytes]:
    """a Record's pair key ('_' + name) -> (name, LTSV type suffix)"""
    name = key[1:]
    if src == LTSV:
        for t, suf in SUFFIXES.items():
            s = suf.encode()
            if name.endswith(s) and TYPED.get(name[:-len(s)].decode("latin-1")) == t:
                return name[:-len(s)], s
    return name, b""


class _Watched(O._Message):
    """the oracle's message, with every allocation and the pointer that reaches it logged"""

    def __init__(self):
        super().__init__()
        self.log = []

    def point(self, ps, pw, place, kind, hi):
        super().point(ps, pw, place, kind, hi)
        self.log.append((ps, pw, place, kind, hi))


def model(rec: dict, extra: list[tuple[bytes, bytes]], src: int = R5):
    """build_capnp's segment list of one record: ([(kind, bytes)], [(message segment, index of the tag, index of the
    last word)] of each pair list, the number of message segments, the allocation log).  Kinds: 'table', 'root', 'data',
    'rptr' (a Record pointer), 'pad', 'tag', 'pw0' / 'pw1' (a pair's data words), 'kptr' / 'vptr' (its pointers), 'us'
    (a pair key's '_'), 'suffix' (an LTSV type suffix), 'end' (the NUL and zero pad), 'body:<where>' (host, app, proc,
    msgid, msg, full, sdid, key, value, xkey, xvalue) and 'json' (a GELF string that held escapes).  An empty body pushes
    nothing; 'end' is always pushed.  Each object's message segment comes from the oracle's allocation log."""
    m = _Watched()
    msg = O.encode(rec, extra, m)
    # the objects in allocation order: ('root',) / ('text', where, body, us, suffix) / ('list', n)
    objs = [("root",)]
    for name in O.FIELDS:
        if rec[name] is not None:
            objs.append(("text", name, rec[name], False, b""))
    if rec["sd"] is not None:
        sd_id, pairs = rec["sd"][0]
        if sd_id is not None:
            objs.append(("text", "sdid", sd_id, False, b""))
        objs.append(("list", len(pairs)))
        for k, (member, v) in pairs:
            name, suf = _key(src, k)
            objs.append(("text", "key", name, True, suf))
            if member == "string":
                objs.append(("text", "value", v, False, b""))
    if extra:
        objs.append(("list", len(extra)))
        for k, v in extra:
            objs += [("text", "xkey", k, False, b""), ("text", "xvalue", v, False, b"")]
    assert len(objs) == len(m.log)
    word = lambda s, i: struct.pack("<Q", m.words[s][i])
    nseg = len(m.size)
    out = [("table", msg[8 * t:8 * t + 8]) for t in range(nseg // 2 + 1)]
    spans = []
    for s in range(nseg):
        if s == 0:
            out += [("root", word(0, 0)), ("data", word(0, 1)), ("data", word(0, 2))]
            out += [("rptr", word(0, 3 + k)) for k in range(9)]
        for obj, (_, _, (os_, pos, pad), _, _) in zip(objs, m.log):
            if os_ != s or obj[0] == "root":
                continue
            if pad is not None:
                out.append(("pad", word(s, pad)))
            if obj[0] == "list":
                n = obj[1]
                out.append(("tag", word(s, pos)))
                first = len(out) - 1
                for j in range(n):
                    out += [(k, word(s, pos + 1 + 4 * j + w)) for w, k in enumerate(("pw0", "pw1", "kptr", "vptr"))]
                spans.append((s, first, len(out) - 1))
                continue
            _, where, body, us, suf = obj
            if us:
                out.append(("us", b"_"))
            if body:
                out.append(("json" if src == GELF and where in ("host", "msg", "full", "key", "value") and _json(body)
                            else "body:" + where, body))
            if suf:
                out.append(("suffix", suf))
            done = sum(len(b) for _, b in out)
            out.append(("end", b"\0" * (8 - done % 8)))
    return out, spans, nseg, m


def segments(rec: dict, extra: list[tuple[bytes, bytes]], src: int = R5) -> list[tuple[str, bytes]]:
    """the (kind, bytes) entries build_capnp pushes for a record, in order (model's first result)"""
    return model(rec, extra, src)[0]


def cells(rec: dict, extra, src: int) -> tuple[set, int, set]:
    """(the (boundary, kind) cells a record reaches, its entry total, the (boundary, list segment) cells of an entry right
    after a whole pair list)"""
    out, spans, _, _ = model(rec, extra, src)
    got = {(b, out[b][0]) for b in BOUNDARIES if b < len(out)}
    after = {(last + 1, s) for s, _, last in spans if last + 1 in (WINDOW, 2 * WINDOW) and last + 1 < len(out)}
    return got, len(out), after


# ---- lines ------------------------------------------------------------------------------------------------------------

def r5_line(values: list[bytes], host: bytes = b"h", msg: bytes | None = b"m", elems: bytes = b"") -> bytes:
    sd = b"[e " + b" ".join(b"n%02d=\"%s\"" % (k, v) for k, v in enumerate(values)) + b"]" if values else b"-"
    return b"<13>1 " + TS + b" " + host + b" a p id " + sd + elems + (b"" if msg is None else b" " + msg)


def ltsv_line(parts: list[bytes], host: bytes = b"h", msg: bytes | None = b"m") -> bytes:
    return b"\t".join([b"time:1438790025.5", b"host:" + host] + parts + [b"level:3"] +
                      ([] if msg is None else [b"message:" + msg]))


def gelf_line(members: list[bytes], host: bytes = b"h", msg: bytes = b"m", full: bool = True) -> bytes:
    return (b'{"host":"' + host + b'","short_message":"' + msg + b'",' + (b'"full_message":"f",' if full else b"") +
            b'"level":3,"timestamp":1.5' + b"".join(b"," + m for m in members) + b"}")


# per source: a pair with a string value, one with an empty value, the target pairs (every kind a pair can put on a
# boundary: an escaped GELF string, an LTSV suffix, a typed value without a text), and the host / msg variants that
# shift every later entry by one or two
_PAIRS = {
    R5: (lambda k: b'v%d' % k, lambda k: b"", [b"word", b'q\\"x', b"a\tb"]),
    LTSV: (lambda k: b"k%02d:v" % k, lambda k: b"k%02d:" % k,
           [b"counter:18446744073709551615", b"mean:0.5", b"done:true", b"t:a b:c", b"score:-1\tdone:false"]),
    GELF: (lambda k: b'"_k%02d":"v"' % k, lambda k: b'"_k%02d":""' % k,
           [b'"_t":"a\\tb"', b'"_q\\"":1', b'"_t":-9223372036854775808', b'"_t":true', b'"_t":null', b'"_t":"word"']),
}


def _line(src: int, pairs: list[bytes], shift: int, msg: bytes = b"m", host: bytes = b"h", elems: bytes = b"") -> bytes:
    """one record of the window or layout lines; shift 0..3 drops 0..3 entries before the pair list (an empty or a
    missing message, an empty host, no full_message)"""
    if src == R5:  # ("-" is a hostname here)
        return r5_line(pairs, host=host, msg=b"" if shift & 1 else msg, elems=elems)
    if src == LTSV:
        return ltsv_line(pairs, host=b"" if shift & 1 else host, msg=None if shift & 2 else msg)
    return gelf_line(pairs, host=b"" if shift & 1 else host, msg=msg, full=not shift & 2)


def window_lines(src: int) -> list[bytes]:
    """Records of 0..24 pairs, with 0..3 of them with an empty value and one target pair last, and 0..3 entries dropped
    before the pair list: totals run through 63..65, 127..129, 191..193 and every kind of KINDS[src] lands on every
    boundary.  A last pair with a value too large for segment 0 puts its landing pad there.  Then records whose pair
    list is in segment 1 (a host and a message that fill segment 0 first), so that a window starts one entry past a whole
    list in segment 0 and in segment 1."""
    if src == R3:
        return [b"<13>Aug  6 11:15:24 host app: m", b"Aug  6 11:15:24 host app: m", b"<13>Aug  6 11:15:24 host app: "]
    full, empty, targets = _PAIRS[src]
    out = []
    for m in range(0, 25):
        for e in range(min(m, 3) + 1):
            for t in targets + [None, _BIG[src]]:
                for shift in range(4):
                    pairs = [empty(k) if k < e else full(k) for k in range(m)] + ([t] if t else [])
                    out.append(_line(src, pairs, shift))
    # the pair list in segment 1: the texts before it take all but a few words of segment 0
    for m in range(1, 33):
        for host, msg, elems in _FILL[src]:
            for shift in range(4):
                out.append(_line(src, [full(k) for k in range(m)], shift, msg=msg, host=host, elems=elems))
    # the extras list in segment 1: a last value (RFC5424: a full_msg) that fills segment 0 all but a few words
    for m in range(0, 20):
        for e in range(min(m, 3) + 1):
            for shift in range(4):
                for w in (0, 6):
                    pairs = [empty(k) if k < e else full(k) for k in range(m)]
                    if src == R5:
                        out.append(_line(src, pairs, shift, elems=b'[big@1 x="' + b"V" * (8 * (980 - 6 * m - w)) + b'"]'))
                        # (a message that fills segment 0, a full_msg in segment 1 before the extras)
                        out.append(_line(src, pairs, 0, msg=b"M" * (8 * (990 - 6 * m - w) - shift)))
                    else:
                        out.append(_line(src, pairs + [_FILLER[src](8 * (990 - 6 * m - w))], shift))
    return out


# a last pair whose value does not fit segment 0; texts that leave the pair list no room there (an RFC5424 full_msg is
# the whole line: a second SD element, never written, makes it long)
_BIG = {R5: b"V" * 8100, LTSV: b"t:" + b"V" * 8100, GELF: b'"_t":"' + b"V" * 8100 + b'"'}
_FILLER = {LTSV: lambda n: b"t:" + b"V" * n, GELF: lambda n: b'"_t":"' + b"V" * n + b'"'}
_FILL = {R5: [(b"h", b"m", b'[big@1 x="' + b"V" * 7950 + b'"]'), (b"h", b"M" * 3900, b"")],
         LTSV: [(b"h", b"M" * 8040, b""), (b"H" * 8040, b"m", b""), (b"H" * 7000, b"M" * 1040, b"")],
         GELF: [(b"h", b"M" * 8040, b""), (b"H" * 8040, b"m", b""), (b"H" * 7000, b"M" * 1040, b"")]}


def layout_lines(src: int) -> dict[str, list[bytes]]:
    """Lines per multi-segment shape, by name:
      - backfill: a pair list too large for segment 0 goes to segment 1; its texts, once segment 1 is full, back-fill
        segment 0, each behind a landing pad there;
      - segment2: ... and once segment 0 is full too, go to a new segment 2;
      - extras: with MANY_EXTRAS, the extras list is larger than any segment left and opens a new one;
      - tables: messages of 3 to 6 segments (texts that each outgrow every segment before them), segment tables of an
        odd and an even number of entries."""
    full = _PAIRS[src][0]
    pair = {R5: lambda k: b"v%d" % k, LTSV: lambda k: b"k%04d:v" % k, GELF: lambda k: b'"_k%04d":"v"' % k}[src]
    big = {R5: lambda k, n: b"v" * n, LTSV: lambda k, n: b"b%d:" % k + b"v" * n,
           GELF: lambda k, n: b'"_b%d":"' % k + b"v" * n + b'"'}[src]
    return {"backfill": [_line(src, [pair(k) for k in range(n)], s) for n in (380, 450, 500) for s in (0, 1)],
            "segment2": [_line(src, [pair(k) for k in range(n)], s) for n in (600, 700) for s in (0, 1)],
            "extras": [_line(src, [full(k) for k in range(n)], 0, msg=b"M" * 7000) for n in (0, 1, 3)],
            "tables": [_line(src, [big(k, 16_000 << k) for k in range(n)], 0) for n in range(1, 6)]}


MANY_EXTRAS = {"x%03d" % k: "v" for k in range(300)}


# lane_lines' records of exactly 64 and 128 entries and of four windows: (pairs, of them with an empty value, shift)
LANE_SHAPES = {R5: {64: (4, 0, 0), 128: (12, 6, 1), 4: (22, 0, 0)}, LTSV: {64: (5, 0, 1), 128: (12, 0, 0), 4: (22, 0, 0)},
               GELF: {64: (5, 0, 1), 128: (12, 0, 0), 4: (22, 0, 0)}}


def lane_line(src: int, n: int, e: int, shift: int) -> bytes:
    full, empty, _ = _PAIRS[src]
    return _line(src, [empty(k) if k < e else full(k) for k in range(n)], shift)


def lane_lines(src: int, rng) -> list[bytes]:
    """Warps of 32 lines: at every lane position, one record of exactly 64 or 128 entries (it ends on a window boundary:
    one more, empty window runs) or of four windows, beside lanes that need one to four windows and one rejected line"""
    if src == R3:
        make = lambda n: b"<13>Aug  6 11:15:24 host app: " + b"x" * (n + 1)
        picks, small = [make(400), make(9000)], [make(k) for k in range(8)]
    else:
        picks = [lane_line(src, *LANE_SHAPES[src][k]) for k in (64, 128, 4)]
        small = [lane_line(src, n, 0, 0) for n in range(0, 23)]
    bad = {R5: b"<13>1 " + TS + b" h a p m [broken", LTSV: b"time:nope\thost:h", GELF: b'{"host":"h"', R3: b"\xff"}[src]
    out = []
    for lane in range(32):
        for big in picks:
            warp = [small[int(x)] for x in rng.integers(0, len(small), 32)]
            warp[lane] = big
            warp[(lane + 7) % 32] = bad
            out += warp
    return out
