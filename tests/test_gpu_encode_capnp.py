"""output.format = "capnp" on the device: the fused Cap'n Proto calls (fg_decode_encode_capnp, fg_split_decode_encode_capnp)
over the four decoders, compared record by record with CapnpEncoder::encode restated over the oracle's Records
(tests/capnp_oracle.py) and read back by the wire-format reader, statuses with fg_decode_batch, output.framing with the
mergers (tests/merger_oracle.py), and the host splitter end to end.  Lines up to 100 KB give messages of several
segments.  GPU only."""
import ctypes as C
import os

import numpy as np
import pytest

import capnp_oracle as O
import merger_oracle as M
import vectors as V
from flowgger_b200.native import FgEncodedOut

pytestmark = pytest.mark.gpu
R5, LTSV, GELF, R3 = 0, 1, 2, 3
YEAR = 2026
INVALID_UTF8 = 76
FG_E_ARG = -1
NTHREADS = os.cpu_count() or 8
TYPED = {"counter": "u64", "score": "i64", "mean": "f64", "done": "bool"}
SUFFIXES = {"u64": "_u64", "i64": "_i64", "f64": "_f64", "bool": "_bool"}
SOURCES = {"rfc5424": R5, "rfc3164": R3, "ltsv": LTSV, "ltsv_typed": LTSV, "gelf": GELF}
SEEDS = {"rfc5424": 15, "rfc3164": 13, "ltsv": 21, "ltsv_typed": 31, "gelf": 12}
EXTRA = {"_x": "a\tb:c", "y:z": "1\n2", "host": "dup", "a": ""}  # keys as given, an empty value
BAD = b"\xff\xfe not UTF-8"

# edge lines per source: several SD elements (only the first is written), an element without pairs, escapes in every
# GELF string, typed values of every kind, empty texts
EDGES = {
    "rfc5424": [b'<13>1 2015-08-05T15:53:45Z h a p m [x@1 a:b="v\tw" a:b="again"][y@2 a:b="3"] msg\twith tab',
                b'<13>1 2015-08-05T15:53:45.1Z - - - - - ',
                b'<13>1 2015-08-05T15:53:45Z h a p m [empty@1][y@2 k="v"] m',
                b'<13>1 2015-08-05T15:53:45Z h a p m [e@1 k="a\\"b\\\\c\\]d"][f@2 k="x"][g@3 k="y"]',
                b'<165>1 2003-10-11T22:14:15.003Z mymachine.example.com evntslog - ID47 [exampleSDID@32473 iut="3" '
                b'eventSource="Application" eventID="1011"] \xef\xbb\xbfAn application event log entry...'],
    "rfc3164": [b"<34>Oct 11 22:14:15 mymachine su: 'su root' failed\tfor lonvick", b"Oct 11 22:14:15 host msg", b"<0>Jan  1 00:00:00 h x"],
    "ltsv": [b"time:1438790025.99\thost:\tmessage:m\tk:v\tk:w", b"time:[2015-08-05T15:53:45Z]\thost:h\tlevel:3\t:x\ta:b:c",
             b"host:h\ttime:1e21\tnovalue\tx:y", b"host:h\ttime:1\tmessage:"],
    "ltsv_typed": [b"time:nan\thost:h\tmean:inf\tcounter:18446744073709551615\tscore:-9223372036854775808",
                   b"time:-0\thost:h\tmean:5e-324\tdone:true\tscore:0", b"time:1e21\thost:h\tmean:-inf\tdone:false\tmean:1e-7",
                   b"time:1438854924.123\thost:h\tmean:-0\tcounter:0"],
    "gelf": [b'{"version":"1.1","host":"h\\tx","short_message":"a\\nb\\t\\u0000c","timestamp":1.5,"_k\\tey":"v\\u00e9","x:y":1e21}',
             b'{"host":"","short_message":"m","_n":null,"_b":true,"_i":-3,"_u":18446744073709551615,"_f":0.1,"timestamp":2}',
             b'{"host":"h","short_message":"no timestamp","_a":"1","a":"2"}',
             b'{"host":"h\\u00e9\\ud83d\\ude00","full_message":"f\\\\n\\"q\\"","level":3,"timestamp":1e-7,"_\\u005fx":"y\\/z"}',
             b'{"host":"h","short_message":"' + b'\\u0041b' * 40 + b'","_\\u006b\\u0065y":"\\"\\\\\\b\\f\\n\\r\\t","timestamp":3}'],
}


def _decoder(native, src, **kw):
    typed = src == "ltsv_typed"
    return native.BatchDecoder(SOURCES[src], ltsv_schema=TYPED if typed else None, ltsv_suffixes=SUFFIXES if typed else None,
                               rfc3164_year=YEAR if src == "rfc3164" else 0, **kw)


def _cfg(oracle, src):
    if src == "rfc3164":
        return oracle.Rfc3164Config(YEAR)
    if src == "ltsv_typed":
        return oracle.LtsvConfig(TYPED, SUFFIXES)
    return None


def _vector_lines(src):
    if src == "rfc5424":
        return [V.G1_LINE, V.G2_LINE] + [l for l, _ in V.RFC5424_CASES]
    if src == "rfc3164":
        return [l for _, _, l, _ in V.RFC3164_GOLDEN] + [l for l, _ in V.RFC3164_CASES]
    if src == "gelf":
        return [V.G3_LINE] + [l for l, _ in V.GELF_CASES]
    return [V.G9_LINE, V.G10_LINE, V.G11_LINE, V.G12_LINE, V.G13_LINE, V.G14_LINE] + [l for l, _ in V.LTSV_CASES] + \
        [l for l, _ in V.LTSV_SCHEMA_CASES]


def _long_lines(src):
    """lines of 4..100 KB: their messages take several segments"""
    out = []
    for k in (4000, 8100, 16_000, 50_000, 100_000):
        if src == "rfc5424":
            out.append(b'<13>1 2015-08-05T15:53:45Z h a p m [x@1 a="' + b"v" * (k // 4) + b'" b="w"][y@2 c="d"] ' + b"m" * k)
        elif src == "rfc3164":
            out.append(b"<13>Oct 11 22:14:15 host tag: " + b"m" * k)
        elif src.startswith("ltsv"):
            out.append(b"host:h\ttime:1.5\tk:" + b"v" * (k // 3) + b"\tmessage:" + b"m" * k + b"\tz:" + b"q" * (k // 5))
        else:
            out.append(b'{"host":"h","short_message":"' + b"m" * k + b'","full_message":"' + b"a\\nb" * (k // 8) +
                       b'","_k":"' + b"v" * (k // 3) + b'","_e":"\\u00e9' * 1 + b'","timestamp":1}')
    return out


def _arr(b: bytes) -> np.ndarray:
    return np.frombuffer(b, dtype=np.uint8).copy() if b else np.zeros(0, np.uint8)


def _pack(lines):
    offs = np.zeros(len(lines) + 1, np.int32)
    np.cumsum([len(l) for l in lines], out=offs[1:])
    return _arr(b"".join(lines)), offs


def _lines(native, src, n):
    """vectors + edges + long lines + n generated lines with decoder rejects; none holds a terminator of either framing"""
    data, offs = native.generate(SOURCES[src], SEEDS[src], n, bad_frac=0.02)
    lines = [l.encode() for l in _vector_lines(src)] + EDGES[src] + _long_lines(src) + \
        [bytes(data[offs[i]:offs[i + 1]]) for i in range(n)]
    return [l for l in lines if b"\n" not in l and b"\r" not in l and b"\0" not in l]


def _records_of(oracle, src, lines, now=None):
    d, o = _pack(lines)
    return O.decode_records(oracle, SOURCES[src], d, o, cfg=_cfg(oracle, src), now=now, nthreads=NTHREADS)


def _expected(oracle, src, lines, extra, now=None):
    ex = O.extra_pairs(extra)
    return [b"" if r is None else O.encode(r, ex) for r in _records_of(oracle, src, lines, now)]


def _records(buf, offs):
    return [buf[offs[i]:offs[i + 1]] for i in range(len(offs) - 1)]


def _first_bad(got, want, lines):
    for i, (g, w) in enumerate(zip(got, want)):
        if g != w:
            return f"record {i} ({len(g)} / {len(w)} bytes): line {lines[i][:200]!r}\n got  {g[:400]!r}\n want {w[:400]!r}"
    return None


@pytest.fixture(scope="module", params=sorted(SOURCES))
def source(request, native):
    src = request.param
    dec = _decoder(native, src, max_batch_bytes=256 << 20, max_batch_lines=1 << 19)
    yield src, dec, _lines(native, src, 200_000)
    dec.close()


def test_prefamed_matches_oracle_and_statuses(source, oracle):
    """every record byte for byte, every record read back to the oracle's Record, statuses as fg_decode_batch's"""
    src, dec, lines = source
    dec.set_capnp_extra(EXTRA)
    d, o = _pack(lines)
    buf, offs, st, _ = dec.decode_encode_capnp(d, o)
    now = dec.gelf_now() if src == "gelf" else None
    recs = _records_of(oracle, src, lines, now)
    ex = O.extra_pairs(EXTRA)
    want = [b"" if r is None else O.encode(r, ex) for r in recs]
    got = _records(buf, offs)
    assert (msg := _first_bad(got, want, lines)) is None, msg
    for g, r in zip(got, recs):
        if r is not None:
            assert O.read(g) == (O.as_read(r), ex)
    assert any(len(g) > 9000 for g in got)  # messages of several segments went through the device
    assert np.array_equal(st, dec.decode(d, o).status.astype(np.uint8))
    assert [bool(w) for w in want] == [s == 0 for s in st]
    if src.startswith("ltsv"):  # the GELF call's "Missing value" stops
        stops = dec.ltsv_stops()
        dec.decode_encode_gelf(d, o)
        assert np.array_equal(stops, dec.ltsv_stops())
    dec.set_capnp_extra({})


@pytest.mark.parametrize("framing", ["line", "nul"])
def test_split_matches_prefamed(source, framing):
    """the raw-stream call: the same records as the pre-framed one, and a record that is not UTF-8 is rejected"""
    src, dec, lines = source
    d, o = _pack(lines)
    pre, po, pst, _ = dec.decode_encode_capnp(d, o)
    delim = b"\n" if framing == "line" else b"\0"
    parts, which = [], []
    for i, l in enumerate(lines):
        if i % 997 == 500:
            parts.append(BAD)
            which.append(None)
        parts.append(l)
        which.append(i)
    buf, offs, st, _, _ = dec.split_decode_encode_capnp(_arr(delim.join(parts) + delim), 0 if framing == "line" else 1)
    got = _records(buf, offs)
    want_pre = _records(pre, po)
    assert len(got) == len(which)
    for j, i in enumerate(which):
        if i is None:
            assert st[j] == INVALID_UTF8 and got[j] == b""
        elif src != "gelf" or pst[i] != 0 or b'"timestamp"' in lines[i]:  # a clock-stamped GELF record differs in ts
            assert got[j] == want_pre[i], (lines[i], got[j], want_pre[i])
            assert st[j] == pst[i]


@pytest.mark.parametrize("out", [M.NONE, M.LINE, M.NUL, M.SYSLEN])
def test_output_framing(source, oracle, out):
    src, dec, lines = source
    lines = lines[:20_000]
    d, o = _pack(lines)
    dec.set_output_framing(out)
    try:
        buf, offs, st, _ = dec.decode_encode_capnp(d, o)
    finally:
        dec.set_output_framing(M.NONE)
    now = dec.gelf_now() if src == "gelf" else None
    want = _expected(oracle, src, lines, None, now)
    assert buf == M.output_stream(want, [s == 0 for s in st], out)
    got = _records(buf, offs)
    for i, w in enumerate(want):
        assert got[i] == (M.MERGERS[out](w) if st[i] == 0 else b"")


def test_gelf_wall_clock(native):
    """a GELF record without "timestamp" gets the wall clock of the call"""
    dec = _decoder(native, "gelf")
    d, o = _pack([b'{"host":"h","short_message":"m"}'])
    buf, _, st, _ = dec.decode_encode_capnp(d, o)
    rec, _ = O.read(buf)
    assert st[0] == 0 and rec["ts_bits"] == int(np.array([dec.gelf_now()], np.float64).view(np.uint64)[0])
    dec.close()


def test_multi_chunk_and_regrow(native, oracle):
    """small chunk_lines (many parse steps) and a context whose output buffer and side tables must grow"""
    for src in ("rfc5424", "gelf", "ltsv_typed"):
        lines = _lines(native, src, 30_000)
        dec = _decoder(native, src, chunk_lines=1000, max_batch_bytes=64 << 20, max_batch_lines=1 << 16)
        d, o = _pack(lines)
        buf, offs, st, _ = dec.decode_encode_capnp(d, o)
        now = dec.gelf_now() if src == "gelf" else None
        want = _expected(oracle, src, lines, None, now)
        assert (msg := _first_bad(_records(buf, offs), want, lines)) is None, msg
        # long extras: every record grows by 60 KB and takes a second segment, past the output buffer of the first call
        big = {"k%02d" % j: "v" * 3000 for j in range(20)}
        dec.set_capnp_extra(big)
        buf, offs, st, _ = dec.decode_encode_capnp(d[:o[2000]].copy(), o[:2001].copy())
        now = dec.gelf_now() if src == "gelf" else None
        want = _expected(oracle, src, lines[:2000], big, now)
        assert (msg := _first_bad(_records(buf, offs), want, lines)) is None, msg
        dec.close()


def test_three_chunk_stream(native):
    """a raw stream of three 64 MiB chunks: the records of the pre-framed call on the same lines"""
    dec = _decoder(native, "rfc5424", max_batch_bytes=200 << 20, max_batch_lines=1 << 21)
    data, offs = native.generate(R5, 77, 1_050_000, terminated=True)
    assert len(data) > 128 << 20
    buf, eo, st, lo, _ = dec.split_decode_encode_capnp(data)
    assert np.array_equal(lo, offs)
    lines, loffs = native.generate(R5, 77, 1_050_000)  # the same lines without their '\n'
    pbuf, peo, pst, _ = dec.decode_encode_capnp(lines, loffs)
    assert np.array_equal(st, pst) and np.array_equal(eo, peo) and buf == pbuf
    assert (st == 0).mean() > 0.9
    dec.close()


def test_extra_arguments(native):
    dec = _decoder(native, "rfc5424")
    L = dec.L
    keys = (C.c_char_p * 2)(b"a", b"a")
    vals = (C.c_char_p * 2)(b"1", b"2")
    dec.set_capnp_extra({"k": "v"})
    assert L.fg_set_capnp_extra(dec.ctx, 2, keys, vals) == FG_E_ARG  # duplicate key
    vals2 = (C.c_char_p * 2)(b"1", None)
    keys2 = (C.c_char_p * 2)(b"a", b"b")
    assert L.fg_set_capnp_extra(dec.ctx, 2, keys2, vals2) == FG_E_ARG  # NULL value
    d, o = _pack([V.G1_LINE.encode()])
    buf, _, _, _ = dec.decode_encode_capnp(d, o)
    assert O.read(buf)[1] == [(b"k", b"v")]  # unchanged by the refused calls
    dec.close()


@pytest.mark.parametrize("src", ["rfc5424", "ltsv", "gelf"])
def test_batching_line_splitter(native, oracle, src):
    """BatchingLineSplitter with CudaCapnpEncoder through the host layer: one message per record, unframed by default"""
    lines = _lines(native, src, 5000)
    dec = _decoder(native, src)
    text = b"\n".join(lines) + b"\n"
    out, err, std = native.splitter_run_capnp_framed(dec, text, extra={"e": "x"}, max_lines=1000)
    g_out, g_err, g_std = native.splitter_run_gelf_framed(dec, text, M.LINE, max_lines=1000)
    now = dec.gelf_now() if src == "gelf" else None
    if src != "gelf":
        assert out == b"".join(_expected(oracle, src, lines, {"e": "x"}, now))
    else:  # the wall clock differs between the batches of the splitter: read the stream back message by message
        n, at = 0, 0
        while at < len(out):
            nseg = int.from_bytes(out[at:at + 4], "little") + 1
            sizes = np.frombuffer(out[at + 4:at + 4 + 4 * nseg], np.uint32)
            size = 8 * (nseg // 2 + 1) + 8 * int(sizes.sum())
            O.read(out[at:at + size])
            at, n = at + size, n + 1
        assert at == len(out) and n == sum(1 for r in _records_of(oracle, src, lines, 0.0) if r is not None)
    assert err == g_err and std == g_std
    dec.close()


def test_text_too_long(native):
    """a text of 2^29 - 1 bytes (capnp-rust asserts on it): the call fails with FG_E_ARG naming the record"""
    dec = _decoder(native, "rfc5424", max_batch_bytes=(1 << 29) + (1 << 20), max_batch_lines=1 << 10)
    head = b"<13>1 2015-08-05T15:53:45Z h a p m - "
    long_line = head + b"m" * ((1 << 29) - 1 - len(head))  # full_msg is the whole line
    ok = V.G1_LINE.encode()
    d, o = _pack([ok, long_line, ok])
    out = FgEncodedOut()
    rc = dec.L.fg_decode_encode_capnp(dec.ctx, R5, d.ctypes.data, o.ctypes.data, 3, C.byref(out))
    assert rc == FG_E_ARG
    assert b"record 1" in dec.L.fg_last_error(dec.ctx)
    d, o = _pack([ok, long_line[:-1], ok])  # one byte less: a message of two segments of 512 MiB texts
    buf, offs, st, _ = dec.decode_encode_capnp(d, o)
    rec, _ = O.read(_records(buf, offs)[1])
    assert list(st) == [0, 0, 0] and rec["full"] == long_line[:-1] and rec["msg"] == long_line[len(head):-1]
    dec.close()
