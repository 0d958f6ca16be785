"""CapnpEncoder::encode (src/flowgger/encoder/capnp_encoder.rs:36-109) restated over the oracle's decoded Records, for the
tests of the fused Cap'n Proto encoder, and a reader of the messages written from the wire format alone.

The encoder builds record.capnp's Record as capnp-rust 0.14's Builder::new_default() does and serializes it as
capnp::serialize::write_message: objects in build_record's order, each first tried in the segment holding its pointer,
else n + 1 words (landing pad + object) in the first segment with room or in a new one of max(n + 1, next_size) words
(next_size from 2048, grown by each new segment's size).  It is pinned to the reference's three encoder tests
(tests/golden/capnp_encoder_tests.json).  The reader follows struct, list and far pointers and rebuilds the Record: a
second check on every message that does not rest on the allocator restated here.

A Record here is a dict: ts_bits (u64 of the f64), fac / sev (int or None), host (bytes), app / proc / msgid / msg / full
(bytes or None), sd (None or a list of (id bytes or None, [(key bytes, (member, value))])), member one of "string"
(bytes), "bool" (bool), "f64" (u64 bits), "i64", "u64" (int), "null" (None)."""
from __future__ import annotations

import struct

from ltsv_oracle import _Reader

SEG0_WORDS = 1024
NEXT_WORDS = 2048
MEMBERS = ("string", "bool", "f64", "i64", "u64", "null")
FIELDS = ("host", "app", "proc", "msgid", "msg", "full")


class _Message:
    def __init__(self):
        self.size = [SEG0_WORDS]
        self.words = [[0]]  # the root pointer
        self.next = NEXT_WORDS

    def alloc(self, p: int, n: int):
        """n words for an object whose pointer is in segment p -> (segment, word, landing pad word or None)"""
        if len(self.words[p]) + n <= self.size[p]:
            at = len(self.words[p])
            self.words[p].extend([0] * n)
            return p, at, None
        m = n + 1
        for s in range(len(self.size)):
            if len(self.words[s]) + m <= self.size[s]:
                break
        else:
            sz = max(m, self.next)
            self.size.append(sz)
            self.words.append([])
            self.next += sz
            s = len(self.size) - 1
        at = len(self.words[s])
        self.words[s].extend([0] * m)
        return s, at + 1, at

    def point(self, ps: int, pw: int, place, kind: int, hi: int) -> None:
        s, pos, pad = place
        if pad is None:
            self.words[ps][pw] = (((pos - pw - 1) << 2) & 0xFFFFFFFF) | kind | (hi << 32)
        else:
            self.words[ps][pw] = 2 | (pad << 3) | (s << 32)
            self.words[s][pad] = kind | (hi << 32)

    def text(self, ps: int, pw: int, b: bytes) -> None:
        n = (len(b) + 8) // 8
        place = self.alloc(ps, n)
        self.point(ps, pw, place, 1, 2 | ((len(b) + 1) << 3))
        s, pos, _ = place
        padded = b + b"\0" * (8 * n - len(b))
        self.words[s][pos:pos + n] = list(struct.unpack(f"<{n}Q", padded))

    def pairs(self, ps: int, pw: int, pairs) -> None:
        n = len(pairs)
        place = self.alloc(ps, 1 + 4 * n)
        self.point(ps, pw, place, 1, 7 | ((4 * n) << 3))
        s, pos, _ = place
        self.words[s][pos] = (n << 2) | ((2 | (2 << 16)) << 32)
        for j, (key, (member, value)) in enumerate(pairs):
            at = pos + 1 + 4 * j
            self.text(s, at + 2, key)
            d = MEMBERS.index(member)
            self.words[s][at] = d | ((1 << 16) if member == "bool" and value else 0)
            if member in ("f64", "u64"):
                self.words[s][at + 1] = value
            elif member == "i64":
                self.words[s][at + 1] = value & 0xFFFFFFFFFFFFFFFF
            elif member == "string":
                self.text(s, at + 3, value)

    def serialize(self) -> bytes:
        n = len(self.size)
        table = struct.pack(f"<{n + 1}I", n - 1, *[len(w) for w in self.words])
        table += b"\0" * (-len(table) % 8)
        return table + b"".join(struct.pack(f"<{len(w)}Q", *w) for w in self.words)


def encode(rec: dict, extra: list[tuple[bytes, bytes]], message: _Message | None = None) -> bytes:
    """capnp_encoder.rs:47-109 + write_message over one Record; extra = output.capnp_extra in table order.  `message`: a
    _Message (or a subclass that watches the allocations) to build into."""
    m = _Message() if message is None else message
    m.point(0, 0, m.alloc(0, 11), 0, 2 | (9 << 16))
    m.words[0][1] = rec["ts_bits"]
    fac, sev = rec["fac"], rec["sev"]
    m.words[0][2] = (0xFF if fac is None else fac) | ((0xFF if sev is None else sev) << 8)
    for k, name in enumerate(FIELDS):
        if rec[name] is not None:
            m.text(0, 3 + k, rec[name])
    if rec["sd"] is not None:
        sd_id, pairs = rec["sd"][0]
        if sd_id is not None:
            m.text(0, 3 + 6, sd_id)
        m.pairs(0, 3 + 7, pairs)
    if extra:
        m.pairs(0, 3 + 8, [(k, ("string", v)) for k, v in extra])
    return m.serialize()


def read(msg: bytes) -> tuple[dict, list[tuple[bytes, bytes]]]:
    """A message -> (its Record, with sd holding the one element a message carries, and its extras).  Written from the
    encoding spec: segment table, struct / list / far pointers, Text as a NUL-terminated byte list."""
    nseg = struct.unpack_from("<I", msg, 0)[0] + 1
    sizes = struct.unpack_from(f"<{nseg}I", msg, 4)
    at = 4 + 4 * nseg
    at += -at % 8
    starts = []
    for sz in sizes:
        starts.append(at)
        at += 8 * sz
    assert at == len(msg), (at, len(msg))

    def word(s, i):
        assert 0 <= i < sizes[s], (s, i, sizes[s])
        return struct.unpack_from("<Q", msg, starts[s] + 8 * i)[0]

    def target(s, i):
        """pointer at word i of segment s -> (segment, first word, kind, upper half), or None for a null pointer"""
        w = word(s, i)
        if w == 0:
            return None
        kind = w & 3
        if kind == 2:
            assert not (w >> 2) & 1, "double-far"
            s, i = w >> 32, (w >> 3) & 0x1FFFFFFF
            w = word(s, i)
            kind = w & 3
            assert kind in (0, 1)
        off = (w & 0xFFFFFFFF) >> 2
        off -= (1 << 30) if off >> 29 else 0
        return s, i + 1 + off, kind, w >> 32

    def text(s, i):
        t = target(s, i)
        if t is None:
            return None
        s, pos, kind, hi = t
        assert kind == 1 and hi & 7 == 2, hex(hi)
        n = hi >> 3
        b = msg[starts[s] + 8 * pos:starts[s] + 8 * pos + n]
        assert len(b) == n and b[-1:] == b"\0"
        return b[:-1]

    def pair_list(s, i):
        t = target(s, i)
        if t is None:
            return None
        s, pos, kind, hi = t
        assert kind == 1 and hi & 7 == 7
        tag = word(s, pos)
        n = (tag & 0xFFFFFFFF) >> 2
        assert tag & 3 == 0 and tag >> 32 == (2 | (2 << 16)) and 4 * n == hi >> 3
        out = []
        for j in range(n):
            e = pos + 1 + 4 * j
            w0 = word(s, e)
            member = MEMBERS[w0 & 0xFFFF]
            value = {"string": lambda: text(s, e + 3), "bool": lambda: bool((w0 >> 16) & 1), "f64": lambda: word(s, e + 1),
                     "i64": lambda: struct.unpack("<q", struct.pack("<Q", word(s, e + 1)))[0], "u64": lambda: word(s, e + 1),
                     "null": lambda: None}[member]()
            out.append((text(s, e + 2), (member, value)))
        return out

    s, pos, kind, hi = target(0, 0)
    assert kind == 0 and hi == 2 | (9 << 16)
    d1 = word(s, pos + 1)
    rec = {"ts_bits": word(s, pos), "fac": None if d1 & 0xFF == 0xFF else d1 & 0xFF,
           "sev": None if (d1 >> 8) & 0xFF == 0xFF else (d1 >> 8) & 0xFF}
    for k, name in enumerate(FIELDS):
        rec[name] = text(s, pos + 2 + k)
    sd_id, pairs = text(s, pos + 2 + 6), pair_list(s, pos + 2 + 7)
    rec["sd"] = None if pairs is None else [(sd_id, pairs)]
    extra = pair_list(s, pos + 2 + 8) or []
    return rec, [(k, v) for k, (_, v) in extra]


def as_read(rec: dict) -> dict:
    """the Record a reader gets back from encode(rec): only the first SD element is written"""
    out = dict(rec)
    if rec["sd"] is not None:
        out["sd"] = rec["sd"][:1]
    return out


def _value(r: _Reader):
    t = r.b[r.i:r.i + 1]
    r.i += 1
    if t == b"s":
        return "string", r.s()
    if t == b"b":
        v = r.b[r.i:r.i + 1]
        r.i += 1
        return "bool", v == b"1"
    if t == b"f":
        bits = int(r.b[r.i:r.i + 16], 16)
        r.i += 16
        return "f64", bits
    if t in (b"i", b"u"):
        j = r.i
        if r.b[r.i:r.i + 1] == b"-":
            r.i += 1
        while r.i < len(r.b) and r.b[r.i:r.i + 1].isdigit():
            r.i += 1
        return ("i64" if t == b"i" else "u64"), int(r.b[j:r.i])
    assert t == b"n", t
    return "null", None


def parse_dump(d: bytes, now: float | None = None):
    """One canonical dump (oracle.cpp dump()) -> a Record as above, or None for a decoder error.  The dump grammar is the
    one ltsv_oracle.parse_dump reads; this reader keeps what capnp writes and that one drops: the element ids and the
    raw typed values."""
    if d.startswith(b"E:"):
        return None
    r = _Reader(d)
    r.lit(b"R:ts=")
    if d.startswith(b"now", r.i):
        r.i += 3
        assert now is not None
        ts_bits = struct.unpack("<Q", struct.pack("<d", now))[0]
    else:
        ts_bits = int(d[r.i:r.i + 16], 16)
        r.i += 16
    rec = {"ts_bits": ts_bits}
    r.lit(b";fac=")
    rec["fac"] = r.num()
    r.lit(b";sev=")
    rec["sev"] = r.num()
    r.lit(b";host=")
    rec["host"] = r.s()
    for name in ("app", "proc", "msgid", "msg", "full"):
        r.lit(b";" + name.encode() + b"=")
        rec[name] = r.o()
    r.lit(b";sd=")
    if d[r.i:r.i + 1] == b"~":
        rec["sd"] = None
        return rec
    sds = []
    for _ in range(r.num()):
        r.lit(b"[id=")
        sd_id = r.o()
        r.lit(b";n=")
        pairs = []
        for _ in range(r.num()):
            r.lit(b";k=")
            k = r.s()
            r.lit(b";v=")
            pairs.append((k, _value(r)))
        r.lit(b"]")
        sds.append((sd_id, pairs))
    rec["sd"] = sds
    return rec


def decode_records(oracle, fmt: int, data, offsets, cfg=None, now: float | None = None, nthreads: int = 8) -> list:
    """the oracle's Record of every line (None for a line the decoder rejects)"""
    buf, offs = oracle.decode_dump(fmt, data, offsets, cfg=cfg, nthreads=nthreads)
    return [parse_dump(buf[offs[i]:offs[i + 1]], now) for i in range(len(offs) - 1)]


def extra_pairs(extra: dict[str, str] | None) -> list[tuple[bytes, bytes]]:
    """output.capnp_extra in the order a TOML table iterates it: byte order of the keys"""
    return sorted((k.encode(), v.encode()) for k, v in (extra or {}).items())


def decode_encode_capnp(oracle, fmt: int, data, offsets, extra: dict[str, str] | None = None, cfg=None, now: float | None = None,
                        nthreads: int = 8) -> list[bytes]:
    """decode + CapnpEncoder::encode per line: one message per line, b"" for a line the decoder rejects"""
    ex = extra_pairs(extra)
    return [b"" if rec is None else encode(rec, ex) for rec in decode_records(oracle, fmt, data, offsets, cfg, now, nthreads)]
