"""Lines for the edges of the fused LTSV encoder (test infrastructure, pure Python, no GPU): a model of the segment list
build_ltsv (fg_ltsv_encode.cu) makes of a record, and lines whose records place every kind of segment on the window
boundaries of that list (kMaxLtsvSegs = 56 segments per window, a longer record is rebuilt window by window)."""
from __future__ import annotations

import numpy as np

R5, LTSV, GELF, R3 = 0, 1, 2, 3
WINDOW = 56
# 0-based segment indices around the window boundaries: the last segment of the first and second window and the first
# segment of the second and third
BOUNDARIES = (WINDOW - 1, WINDOW, 2 * WINDOW - 1, 2 * WINDOW)
TOTALS = (55, 56, 57, 111, 112, 113, 167, 168, 169)
TYPED = {"counter": "u64", "score": "i64", "mean": "f64", "done": "bool"}
SUFFIXES = {"u64": "_u64", "i64": "_i64", "f64": "_f64", "bool": "_bool"}
TS = b"2015-08-05T15:53:45.637824Z"
TYPED_NAMES = {k.encode(): v for k, v in TYPED.items()}
# GELF typed values of the lines below as the oracle's Record renders them, and their fg_tag
GELF_NUMBERS = {b"1000000000000000000000": "f64", b"0.5": "f64", b"-9223372036854775808": "i64",
                b"18446744073709551615": "u64", b"true": "bool", b"false": "bool"}
GELF_JSON = {b"a\tb", b'q"x'}  # the unescaped text of the escaped GELF string values below

# the segment kinds each source can put on a window boundary (RFC3164 records have no pairs and never reach one)
_FIXED = {"extras", "field", "host", "num:ts", "msg", "full", "level"}
KINDS = {R5: _FIXED | {"key", "lit", "value", "num:facility", "app", "proc", "msgid"},
         LTSV: _FIXED | {"key", "suffix", "lit", "value", "num:u64", "num:i64", "num:f64", "num:bool"},
         GELF: _FIXED | {"key", "lit", "value", "json", "num:u64", "num:i64", "num:f64", "num:bool"}}


def segments(rec: dict, src: int, extra: bool) -> list[str]:
    """The kinds of the non-empty segments build_ltsv pushes for a Record (as ltsv_oracle.parse_dump gives it), in order:
    'lit' (a pair's tab or ':'), 'key', 'suffix' (LTSV: a typed key's suffix), 'value' (a pair's string), 'json' (a GELF
    string that held escapes), 'num:<type>' (a typed value), 'extras' (the output.ltsv_extra blob), 'field' (a fixed
    field's `\tname:`), and the fixed fields' texts: 'host', 'num:ts', 'msg', 'full', 'level', 'num:facility', 'app',
    'proc', 'msgid'.  An empty name or value pushes nothing; a GELF Null is an empty value."""
    out: list[str] = []
    first = True
    for sd in rec["sd"] or []:
        for name, value in sd:
            if not first:
                out.append("lit")
            first = False
            key = name[1:] if name.startswith(b"_") else name
            typed = None
            if src == LTSV:
                for t, suf in SUFFIXES.items():
                    if key.endswith(suf.encode()) and TYPED_NAMES.get(key[:-len(suf)]) == t:
                        typed = t
            if typed:
                out += ["key", "suffix"]
            elif key:
                out.append("key")
            out.append("lit")
            if typed:
                out.append("num:" + typed)
            elif src == GELF and value in GELF_NUMBERS:
                out.append("num:" + GELF_NUMBERS[value])
            elif value:
                out.append("json" if src == GELF and value in GELF_JSON else "value")
    if extra:
        out.append("extras")

    def field(v, kind, always=False):
        if v is None and not always:
            return
        out.append("field")
        if v:
            out.append(kind)
    field(rec["host"], "host", always=True)
    out += ["field", "num:ts"]
    field(rec["msg"], "msg")
    field(rec["full"], "full")
    if rec["sev"] is not None:
        out += ["field", "level"]
    if rec["fac"] is not None:
        out += ["field", "num:facility"]
    for k in ("app", "proc", "msgid"):
        field(rec[k], k)
    return out


def r5_line(values: list[bytes], host: bytes = b"h", msg: bytes = b"m") -> bytes:
    sd = b"[e " + b" ".join(b"n%02d=\"%s\"" % (k, v) for k, v in enumerate(values)) + b"]" if values else b"-"
    return b"<13>1 " + TS + b" " + host + b" a p id " + sd + b" " + msg


def ltsv_line(parts: list[bytes], host: bytes = b"h") -> bytes:
    return b"\t".join([b"time:1438790025.5", b"host:" + host] + parts + [b"level:3", b"message:m"])


def gelf_line(members: list[bytes], host: bytes = b"h") -> bytes:
    return (b'{"host":"' + host + b'","short_message":"m","full_message":"f","level":3,"timestamp":1.5' +
            b"".join(b"," + m for m in members) + b"}")


# per source: a pair of four segments, one of three (empty value), and the pairs whose segments must reach the
# boundaries.  A line is `e` three-segment and `m - e` four-segment pairs, then one target pair: with m and e swept,
# every segment of the target and of the fixed fields after it lands on every boundary.
_PAIRS = {
    R5: (lambda k: b'n%02d="v"' % k, lambda k: b'n%02d=""' % k,
         [b't="word"', b't="q\\"x"', b't="a\tb:c"']),
    LTSV: (lambda k: b"k%02d:v" % k, lambda k: b"k%02d:" % k,
           [b"counter:18446744073709551615", b"score:-9223372036854775808", b"mean:0.5", b"done:true", b"t:a b:c"]),
    GELF: (lambda k: b'"_k%02d":"v"' % k, lambda k: b'"_k%02d":""' % k,
           [b'"_t":"a\\tb"', b'"_t":"q\\"x"', b'"_t":1e21', b'"_t":-9223372036854775808', b'"_t":18446744073709551615',
            b'"_t":true', b'"_t":null', b'"_t":"word"']),
}


def window_lines(src: int) -> list[bytes]:
    """Records of 0 .. 46 pairs whose segment totals run through 55..57, 111..113, 167..169 and which put every kind of
    KINDS[src] on every boundary; plus the first-field cases: an SD pair with an empty name first, a record without
    pairs (extras or host first), an empty host."""
    if src == R3:
        return [b"<13>Aug  6 11:15:24 host app: m", b"Aug  6 11:15:24 host app: m", b"<13>Aug  6 11:15:24 host app: "]
    four, three, targets = _PAIRS[src]
    out = []
    for m in range(0, 47):
        for e in range(min(m, 3) + 1):
            for t in targets + [None]:
                pairs = [three(k) if k < e else four(k) for k in range(m)] + ([t] if t else [])
                host = b"" if (m + e) % 5 == 0 else b"h"
                if src == R5:
                    sd = b"[e " + b" ".join(pairs) + b"]" if pairs else b"-"
                    out.append(b"<13>1 " + TS + b" " + (host or b"-") + b" a p id " + sd + b" m")
                elif src == LTSV:
                    out.append(ltsv_line(pairs, host=host))
                else:
                    out.append(gelf_line(pairs, host=host))
    if src == LTSV:
        out.append(b"\t".join([b":empty-name", b"time:1.5", b"host:h", b"k:v"]))
    if src == GELF:
        out.append(b'{"_":"noname","host":"h","short_message":"m","_k":"v"}')
    return out


def lane_lines(src: int, rng) -> list[bytes]:
    """Warps of 32 lines: one rejected line and one record of four windows at every lane position; warps whose lanes
    need one to four windows"""
    make = {R5: lambda n: r5_line([b"v%d" % k for k in range(n)]),
            LTSV: lambda n: ltsv_line([b"k%02d:v" % k for k in range(n)]),
            GELF: lambda n: gelf_line([b'"_k%02d":"v"' % k for k in range(n)]),
            R3: lambda n: b"<13>Aug  6 11:15:24 host app: " + b"x" * (n + 1)}[src]
    bad = {R5: b"<13>1 " + TS + b" h a p m [broken", LTSV: b"time:nope\thost:h", GELF: b'{"host":"h"', R3: b"\xff"}[src]
    out = []
    for lane in range(32):
        warp = [make(int(rng.integers(0, 6))) for _ in range(32)]
        warp[lane] = make(45)
        warp[(lane + 7) % 32] = bad
        out += warp
    for _ in range(4):
        out += [make([3, 16, 30, 45][int(x)]) for x in rng.integers(0, 4, 32)]
    return out


def long_lines(src: int, rng) -> list[bytes]:
    """lines of 1008 bytes and more (length class 63) among short ones, with pairs where the source has them"""
    pad = lambda L: bytes(rng.integers(97, 123, L, dtype=np.uint8))
    make = {R5: lambda L: r5_line([b"v"], msg=pad(L)), LTSV: lambda L: ltsv_line([b"k:v"]) + pad(L),
            GELF: lambda L: gelf_line([b'"_k":"%s"' % pad(L)]), R3: lambda L: b"<13>Aug  6 11:15:24 host app: " + pad(L)}[src]
    return [make(1008 + (k % 40) if k % 3 == 0 else int(rng.integers(10, 120))) for k in range(600)]


def span_lines(src: int, rng) -> list[bytes]:
    """20 CTAs of short lines, one of whose 256-line spans is ~140 KB: larger than any encoder tile, read from global"""
    pad = lambda L: bytes(rng.integers(97, 123, L, dtype=np.uint8))
    make = {R5: lambda L: r5_line([b"v"], msg=pad(L)), LTSV: lambda L: ltsv_line([b"k:v"]) + pad(L),
            GELF: lambda L: gelf_line([b'"_k":"%s"' % pad(L)]), R3: lambda L: b"<13>Aug  6 11:15:24 host app: " + pad(L)}[src]
    return [make(int(rng.integers(450, 650)) if 256 * 4 <= k < 256 * 5 else 20) for k in range(256 * 20)]
