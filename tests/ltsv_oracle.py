"""LTSVEncoder::encode (src/flowgger/encoder/ltsv_encoder.rs:66-123) restated over the oracle's decoded Records, for the
tests of the fused LTSV encoder.  The Records come from the oracle's canonical dumps (oracle.decode_dump), so the
decoders are the oracle's; the encoder and Rust's Display for f64 are restated here independently of the device code:
the shortest round-trip digits are Python's repr (David Gay's shortest mode, the same digits as core's
flt2dec::format_shortest), laid out positionally."""
from __future__ import annotations

import math
import struct


def rust_f64(x: float) -> str:
    """`x.to_string()` in Rust: shortest digits that read back to x, positional, no exponent, no trailing ".0"."""
    if math.isnan(x):
        return "NaN"
    if math.isinf(x):
        return "inf" if x > 0 else "-inf"
    if x == 0:
        return "-0" if math.copysign(1.0, x) < 0 else "0"
    r = repr(x)
    neg = r.startswith("-")
    r = r.lstrip("-")
    m, e = (r.split("e") + ["0"])[:2]
    e = int(e)
    ip, fp = (m.split(".") + [""])[:2]
    digits = (ip + fp).lstrip("0")
    e -= len(fp)
    while digits.endswith("0"):
        digits = digits[:-1]
        e += 1
    if e >= 0:
        t = digits + "0" * e
    elif len(digits) + e > 0:
        t = digits[:len(digits) + e] + "." + digits[len(digits) + e:]
    else:
        t = "0." + "0" * -(len(digits) + e) + digits
    return ("-" if neg else "") + t


def esc_key(k: bytes) -> bytes:
    return k.replace(b"\n", b" ").replace(b"\t", b" ").replace(b":", b"_")


def esc_val(v: bytes) -> bytes:
    return v.replace(b"\t", b" ").replace(b"\n", b" ")


def encode(rec: dict, extra: list[tuple[bytes, bytes]]) -> bytes:
    """ltsv_encoder.rs:66-123 over one Record (as parse_dump gives it); extra = output.ltsv_extra in table order."""
    fields: list[tuple[bytes, bytes]] = []
    for sd in rec["sd"] or []:
        for name, value in sd:
            fields.append((name[1:] if name.startswith(b"_") else name, value))
    for k, v in extra:
        fields.append((k[1:] if k.startswith(b"_") else k, v))
    fields.append((b"host", rec["host"]))
    fields.append((b"time", rust_f64(rec["ts"]).encode()))
    for key, name in ((b"message", "msg"), (b"full_message", "full")):
        if rec[name] is not None:
            fields.append((key, rec[name]))
    for key, name in ((b"level", "sev"), (b"facility", "fac")):
        if rec[name] is not None:
            fields.append((key, str(rec[name]).encode()))
    for key, name in ((b"appname", "app"), (b"procid", "proc"), (b"msgid", "msgid")):
        if rec[name] is not None:
            fields.append((key, rec[name]))
    return b"\t".join(esc_key(k) + b":" + esc_val(v) for k, v in fields)


class _Reader:
    def __init__(self, b: bytes):
        self.b, self.i = b, 0

    def lit(self, s: bytes) -> None:
        assert self.b.startswith(s, self.i), (self.b[self.i:self.i + 40], s)
        self.i += len(s)

    def until(self, c: bytes) -> bytes:
        j = self.b.index(c, self.i)
        v, self.i = self.b[self.i:j], j
        return v

    def s(self) -> bytes:  # put_s: "<len>:" + bytes
        n = int(self.until(b":"))
        self.i += 1
        v = self.b[self.i:self.i + n]
        self.i += n
        return v

    def o(self):  # put_o: '~' or put_s
        if self.b[self.i:self.i + 1] == b"~":
            self.i += 1
            return None
        return self.s()

    def num(self):
        if self.b[self.i:self.i + 1] == b"~":
            self.i += 1
            return None
        j = self.i
        while self.i < len(self.b) and self.b[self.i:self.i + 1].isdigit():
            self.i += 1
        return int(self.b[j:self.i])


def _value(r: _Reader) -> bytes:
    t = r.b[r.i:r.i + 1]
    r.i += 1
    if t == b"s":
        return r.s()
    if t == b"b":
        v = r.b[r.i:r.i + 1]
        r.i += 1
        return b"true" if v == b"1" else b"false"
    if t == b"f":
        bits = int(r.b[r.i:r.i + 16], 16)
        r.i += 16
        return rust_f64(struct.unpack("<d", struct.pack("<Q", bits))[0]).encode()
    if t in (b"i", b"u"):
        j = r.i
        if r.b[r.i:r.i + 1] == b"-":
            r.i += 1
        while r.i < len(r.b) and r.b[r.i:r.i + 1].isdigit():
            r.i += 1
        return r.b[j:r.i]
    assert t == b"n", t
    return b""


def parse_dump(d: bytes, now: float | None = None):
    """One canonical dump (oracle.cpp dump()) -> a Record dict, or None for a decoder error.  A GELF Record stamped with
    the wall clock ("ts=now") gets `now`."""
    if d.startswith(b"E:"):
        return None
    r = _Reader(d)
    r.lit(b"R:ts=")
    if d.startswith(b"now", r.i):
        r.i += 3
        assert now is not None
        ts = now
    else:
        ts = struct.unpack("<d", struct.pack("<Q", int(d[r.i:r.i + 16], 16)))[0]
        r.i += 16
    rec = {"ts": ts}
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
    n_sd = r.num()
    sds = []
    for _ in range(n_sd):
        r.lit(b"[id=")
        r.o()
        r.lit(b";n=")
        pairs = []
        for _ in range(r.num()):
            r.lit(b";k=")
            k = r.s()
            r.lit(b";v=")
            pairs.append((k, _value(r)))
        r.lit(b"]")
        sds.append(pairs)
    rec["sd"] = sds
    return rec


def decode_encode_ltsv(oracle, fmt: int, data, offsets, extra: dict[str, str] | None = None, cfg=None, now: float | None = None,
                       nthreads: int = 8) -> list[bytes]:
    """decode + LTSVEncoder::encode per line: one record per line, b"" for a line the decoder rejects.  extra =
    output.ltsv_extra (written in byte order of the keys, as a TOML table iterates)."""
    buf, offs = oracle.decode_dump(fmt, data, offsets, cfg=cfg, nthreads=nthreads)
    ex = sorted((k.encode(), v.encode()) for k, v in (extra or {}).items())
    out = []
    for i in range(len(offs) - 1):
        rec = parse_dump(buf[offs[i]:offs[i + 1]], now)
        out.append(b"" if rec is None else encode(rec, ex))
    return out
