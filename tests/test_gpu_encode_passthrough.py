"""output.format = "passthrough" on the device: the fused passthrough calls (fg_decode_encode_passthrough,
fg_split_decode_encode_passthrough) over the four decoders, compared record by record with PassthroughEncoder::encode
restated over the oracle's Records (tests/passthrough_oracle.py): the header, then Record.full_msg.  Statuses are
fg_decode_batch's, plus FG_EP_NO_RAW exactly where a GELF object has no full_message; output.framing is checked with
the mergers (tests/merger_oracle.py), and the host splitter end to end.  GPU only."""
import os

import numpy as np
import pytest

import merger_oracle as M
import passthrough_oracle as O
import vectors as V
from test_emu_ltsv_json import RETRY

pytestmark = pytest.mark.gpu
R5, LTSV, GELF, R3 = 0, 1, 2, 3
YEAR = 2026
INVALID_UTF8 = 76
NO_RAW = O.FG_EP_NO_RAW
FG_E_ARG = -1
NTHREADS = os.cpu_count() or 8
TYPED = {"counter": "u64", "score": "i64", "mean": "f64", "done": "bool"}
SUFFIXES = {"u64": "_u64", "i64": "_i64", "f64": "_f64", "bool": "_bool"}
SOURCES = {"rfc5424": R5, "rfc3164": R3, "ltsv": LTSV, "ltsv_typed": LTSV, "gelf": GELF}
SEEDS = {"rfc5424": 15, "rfc3164": 13, "ltsv": 21, "ltsv_typed": 31, "gelf": 12}
HEADER = b"[2026-10-18T12:34:56Z] "
BAD = b"\xff\xfe not UTF-8"
GELF_ESCAPES = b'\\"\\\\\\/\\b\\f\\n\\r\\t\\u00e9\\u0000\\ud83d\\ude00\\u20ac'

# edge lines per source: trailing white space (trimmed by RFC5424 and RFC3164, kept by LTSV), a BOM, every GELF escape,
# full_message "", absent and not a string
EDGES = {
    "rfc5424": [b"\xef\xbb\xbf<13>1 2015-08-05T15:53:45Z h a p m - bom line",
                b"<13>1 2015-08-05T15:53:45Z h a p m - trailing tab\t",
                b"<13>1 2015-08-05T15:53:45Z h a p m - nbsp \xc2\xa0 and ideographic \xe3\x80\x80",
                b"<13>1 2015-08-05T15:53:45Z h a p m [x@1 k=\"v\"]  \t \xe3\x80\x80\xc2\xa0",
                b"<13>1 2015-08-05T15:53:45.1Z - - - - - "],
    "rfc3164": [b"<34>Oct 11 22:14:15 mymachine su: 'su root' failed   \t ", b"Oct 11 22:14:15 host msg  ",
                b"<0>Jan  1 00:00:00 h x\xc2\xa0"],
    "ltsv": [b"host:h\ttime:1\tmessage:trailing spaces   ", b"time:1438790025.99\thost:\tmessage:m\tk:v\tk:w \t",
             b"host:h\ttime:1e21\tnovalue\tx:y"],
    "ltsv_typed": [b"time:nan\thost:h\tmean:inf\tcounter:18446744073709551615  ", b"time:-0\thost:h\tdone:true\tscore:0"],
    "gelf": [b'{"host":"h","short_message":"m","full_message":"' + GELF_ESCAPES + b'","timestamp":1}',
             b'{"host":"h","short_message":"m","full_message":"","timestamp":1}',
             b'{"host":"h","short_message":"m","timestamp":1}',
             b'{"host":"h","short_message":"m","full_message":3,"timestamp":1}',
             b'{"host":"h","full_message":"x' + b"\\u0041b" * 40 + b'","timestamp":2}',
             b'{"host":"h","short_message":"m","full_message":"plain  ","timestamp":2}'],
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
    """lines of 4..100 KB"""
    out = []
    for k in (4000, 8100, 16_000, 50_000, 100_000):
        if src == "rfc5424":
            out.append(b'<13>1 2015-08-05T15:53:45Z h a p m [x@1 a="' + b"v" * (k // 4) + b'"] ' + b"m" * k)
        elif src == "rfc3164":
            out.append(b"<13>Oct 11 22:14:15 host tag: " + b"m" * k)
        elif src.startswith("ltsv"):
            out.append(b"host:h\ttime:1.5\tk:" + b"v" * (k // 3) + b"\tmessage:" + b"m" * k)
        else:
            out.append(b'{"host":"h","short_message":"m","full_message":"' + b"a\\nb" * (k // 8) + b'","timestamp":1}')
            out.append(b'{"host":"h","short_message":"m","full_message":"' + b"q" * k + b'","timestamp":1}')
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


def _expected(oracle, src, lines, header):
    d, o = _pack(lines)
    return O.decode_encode_passthrough(oracle, SOURCES[src], d, o, header, cfg=_cfg(oracle, src), nthreads=NTHREADS)


def _records(buf, offs):
    return [buf[offs[i]:offs[i + 1]] for i in range(len(offs) - 1)]


def _first_bad(got, want, lines):
    for i, (g, w) in enumerate(zip(got, want)):
        if g != w:
            return f"record {i} ({len(g)} / {len(w)} bytes): line {lines[i][:200]!r}\n got  {g[:400]!r}\n want {w[:400]!r}"
    return None


def _check(dec, oracle, src, lines, header):
    """the pre-framed call against the oracle, record by record, and its statuses against fg_decode_batch's"""
    dec.set_passthrough_prefix(header)
    d, o = _pack(lines)
    buf, offs, st, _ = dec.decode_encode_passthrough(d, o)
    want, no_raw = _expected(oracle, src, lines, header)
    assert (msg := _first_bad(_records(buf, offs), want, lines)) is None, msg
    dst = dec.decode(d, o).status.astype(np.uint8)
    assert np.array_equal(st, np.where(no_raw, NO_RAW, dst)), [(lines[i], st[i], dst[i]) for i in np.flatnonzero(st != dst)[:5]]
    return buf, offs, st


@pytest.fixture(scope="module", params=sorted(SOURCES))
def source(request, native):
    src = request.param
    dec = _decoder(native, src, max_batch_bytes=256 << 20, max_batch_lines=1 << 19)
    yield src, dec, _lines(native, src, 200_000)
    dec.close()


def test_prefamed_matches_oracle_and_statuses(source, oracle):
    src, dec, lines = source
    _, _, st = _check(dec, oracle, src, lines, HEADER)
    assert (st == NO_RAW).any() == (src == "gelf")
    if src.startswith("ltsv"):  # the "Missing value" stops of a passthrough call are those of a GELF call
        stops = dec.ltsv_stops()
        d, o = _pack(lines)
        dec.decode_encode_gelf(d, o)
        assert np.array_equal(stops, dec.ltsv_stops())


@pytest.mark.parametrize("header", [b"", b"x", b"a\0b\nc", b"<" * 61], ids=["empty", "short", "nul-lf", "61"])
def test_headers(source, oracle, header):
    src, dec, lines = source
    _check(dec, oracle, src, lines[:20_000], header)


@pytest.mark.parametrize("framing", ["line", "nul"])
def test_split_matches_prefamed(source, framing):
    """the raw-stream call: the same records as the pre-framed one, and a record that is not UTF-8 is rejected"""
    src, dec, lines = source
    dec.set_passthrough_prefix(HEADER)
    d, o = _pack(lines)
    pre, po, pst, _ = dec.decode_encode_passthrough(d, o)
    delim = b"\n" if framing == "line" else b"\0"
    parts, which = [], []
    for i, l in enumerate(lines):
        if i % 997 == 500:
            parts.append(BAD)
            which.append(None)
        parts.append(l)
        which.append(i)
    buf, offs, st, _, _ = dec.split_decode_encode_passthrough(_arr(delim.join(parts) + delim), 0 if framing == "line" else 1)
    got = _records(buf, offs)
    want_pre = _records(pre, po)
    assert len(got) == len(which)
    for j, i in enumerate(which):
        if i is None:
            assert st[j] == INVALID_UTF8 and got[j] == b""
        else:
            assert got[j] == want_pre[i] and st[j] == pst[i], (lines[i], got[j], want_pre[i])


@pytest.mark.parametrize("out", [M.NONE, M.LINE, M.NUL, M.SYSLEN])
def test_output_framing(source, oracle, out):
    """an accepted empty record (GELF full_message "") is framed; a rejected one, NO_RAW included, is not"""
    src, dec, lines = source
    lines = lines[:20_000]
    d, o = _pack(lines)
    dec.set_passthrough_prefix(b"")
    dec.set_output_framing(out)
    try:
        buf, offs, st, _ = dec.decode_encode_passthrough(d, o)
    finally:
        dec.set_output_framing(M.NONE)
    want, _ = _expected(oracle, src, lines, b"")
    assert buf == M.output_stream(want, [s == 0 for s in st], out)
    got = _records(buf, offs)
    for i, w in enumerate(want):
        assert got[i] == (M.MERGERS[out](w) if st[i] == 0 else b"")
    if src == "gelf":
        empty = lines.index(EDGES["gelf"][1])
        assert st[empty] == 0 and got[empty] == M.MERGERS[out](b"")


def test_edge_lines_prefamed(native, oracle):
    """lines no split stream holds: RFC5424 and RFC3164 with "\\r\\n" (trimmed), LTSV with "\\r" (kept), GELF retry lines
    (a raw LF: the decoder's newline retry), also split from a NUL-framed stream"""
    cases = {"rfc5424": [b"<13>1 2015-08-05T15:53:45Z h a p m - crlf\r\n", b"\xef\xbb\xbf<13>1 2015-08-05T15:53:45Z h a p m - m \r\n"],
             "rfc3164": [b"<13>Oct 11 22:14:15 host tag: crlf\r\n"],
             "ltsv": [b"host:h\ttime:1\tmessage:cr\r"],
             "gelf": [b'{"host":"h","short_message":"m","full_message":"' + b + b'","timestamp":1}' for b in RETRY]}
    for src, lines in cases.items():
        dec = _decoder(native, src)
        buf, offs, st = _check(dec, oracle, src, lines, HEADER)
        if src == "gelf":
            assert (st == 0).sum() >= 2 * len(lines) // 3
            sbuf, soffs, sst, _, _ = dec.split_decode_encode_passthrough(_arr(b"\0".join(lines) + b"\0"), 1)
            assert np.array_equal(sst, st) and sbuf == buf and np.array_equal(soffs, offs)
        dec.close()


def test_record_lengths(native, oracle):
    """records of 0 bytes to 100 KB: GELF full_message of every length 0..600 with and without escapes, then longer"""
    lens = list(range(601)) + [4095, 4096, 65535, 65536, 100_000]
    lines = []
    for k in lens:
        lines.append(b'{"host":"h","short_message":"m","full_message":"' + (b"abcdefghi" * (k // 9 + 1))[:k] + b'","timestamp":1}')
        lines.append(b'{"host":"h","short_message":"m","full_message":"' + (b"ab\\tc" * (k // 5 + 1))[:k].rstrip(b"\\") + b'","timestamp":1}')
    dec = _decoder(native, "gelf")
    for header in (b"", b"hdr"):
        buf, offs, st = _check(dec, oracle, "gelf", lines, header)
        assert (st == 0).all()
    assert int(np.diff(offs).min()) == 3 and int(np.diff(offs).max()) == 100_003
    dec.close()


def test_multi_chunk_and_regrow(native, oracle):
    """small chunk_lines (many parse steps) and a context whose output buffer must grow for a long header"""
    for src in ("rfc5424", "gelf", "ltsv_typed"):
        lines = _lines(native, src, 30_000)
        dec = _decoder(native, src, chunk_lines=1000, max_batch_bytes=64 << 20, max_batch_lines=1 << 16)
        _check(dec, oracle, src, lines, HEADER)
        # a 60 KB header: 2000 records pass the output buffer of the first call
        _check(dec, oracle, src, lines[:2000], b"h" * 60_000)
        dec.close()


def test_three_chunk_stream(native):
    """a raw stream of three 64 MiB chunks: the records of the pre-framed call on the same lines"""
    dec = _decoder(native, "rfc5424", max_batch_bytes=200 << 20, max_batch_lines=1 << 21)
    dec.set_passthrough_prefix(HEADER)
    data, offs = native.generate(R5, 77, 1_050_000, terminated=True)
    assert len(data) > 128 << 20
    buf, eo, st, lo, _ = dec.split_decode_encode_passthrough(data)
    assert np.array_equal(lo, offs)
    lines, loffs = native.generate(R5, 77, 1_050_000)  # the same lines without their '\n'
    pbuf, peo, pst, _ = dec.decode_encode_passthrough(lines, loffs)
    assert np.array_equal(st, pst) and np.array_equal(eo, peo) and buf == pbuf
    assert (st == 0).mean() > 0.9
    dec.close()


def test_prefix_arguments(native):
    dec = _decoder(native, "rfc5424")
    L = dec.L
    dec.set_passthrough_prefix(b"keep:")
    small = b"0123"
    assert L.fg_set_passthrough_prefix(dec.ctx, None, 3) == FG_E_ARG  # NULL bytes with n > 0
    assert L.fg_set_passthrough_prefix(dec.ctx, small, 1 << 31) == FG_E_ARG  # 2^31 bytes
    assert L.fg_set_passthrough_prefix(dec.ctx, small, -1) == FG_E_ARG
    line = V.G1_LINE.encode()
    d, o = _pack([line])
    buf, _, _, _ = dec.decode_encode_passthrough(d, o)
    assert buf == b"keep:" + line  # unchanged by the refused calls
    assert L.fg_set_passthrough_prefix(dec.ctx, None, 0) == 0  # n = 0 clears it
    assert dec.decode_encode_passthrough(d, o)[0] == line
    dec.close()


@pytest.mark.parametrize("src", ["rfc5424", "gelf"])
def test_launch_count(native, src):
    """a passthrough call launches what a Cap'n Proto call does: the parse kernels, then size, scan, base and write"""
    dec = _decoder(native, src)
    d, o = _pack([l.encode() for l in _vector_lines(src)])
    deltas = []
    for call in (dec.decode_encode_capnp, dec.decode_encode_passthrough):
        before = dec.L.fg_kernel_launches(dec.ctx)
        call(d, o)
        deltas.append(dec.L.fg_kernel_launches(dec.ctx) - before)
    assert deltas[0] == deltas[1] > 4
    dec.close()


@pytest.mark.parametrize("src", ["rfc5424", "ltsv", "gelf"])
def test_batching_line_splitter(native, oracle, src):
    """BatchingLineSplitter with CudaPassthroughEncoder through the host layer: one record per Ok line; a GELF line
    without full_message prints "Cannot output empty raw message: [line]" on stderr, in stream order, as a decoder
    error does"""
    lines = _lines(native, src, 5000)
    dec = _decoder(native, src)
    text = b"\n".join(lines) + b"\n"
    want, no_raw = _expected(oracle, src, lines, b"H ")
    st = dec.decode(*_pack(lines)).status
    g_out, g_err, g_std = native.splitter_run_gelf_framed(dec, text, M.LINE, max_lines=1000)
    g_lines = iter(g_err.split(b"\n")[:-1])
    want_err = []
    for l, s, n in zip(lines, st, no_raw):  # the GELF run prints one line per decoder error, in stream order
        if s != 0:
            want_err.append(next(g_lines) + b"\n")
        elif n:
            want_err.append(b"Cannot output empty raw message: [" + l.strip() + b"]\n")
    assert next(g_lines, None) is None and (src == "gelf") == any(no_raw)
    for out in (M.NONE, M.LINE):
        stream, err, std = native.splitter_run_passthrough_framed(dec, text, out, header=b"H ", max_lines=1000)
        assert stream == b"".join(M.MERGERS[out](w) for w, s, n in zip(want, st, no_raw) if s == 0 and not n)
        assert err == b"".join(want_err) and std == g_std
    dec.close()


# ---- past 4 GiB of output ------------------------------------------------------------------------------------------

def test_past_4gib(native, oracle):
    """a 64 MiB header over 66 lines: 4.2 GB of output from one launch.  Every offset, every record's header and body,
    and the bytes around each record boundary past 2^32"""
    rng = np.random.default_rng(4)
    header = rng.integers(0, 256, 64 << 20, dtype=np.uint8).tobytes()
    lines = [b"<13>1 2015-08-05T15:53:45Z h a p m - line %d " % i + b"x" * int(rng.integers(0, 300)) for i in range(66)]
    lines[7] = b"not a line"  # rejected: no record
    dec = _decoder(native, "rfc5424", max_batch_bytes=1 << 20, max_batch_lines=1 << 10)
    try:
        dec.set_passthrough_prefix(header)
        d, o = _pack(lines)
        buf, offs, st, _ = dec.decode_encode_passthrough(d, o, copy=False)
        want, _ = _expected(oracle, "rfc5424", lines, b"")
        lens = [0 if s else len(header) + len(w) for w, s in zip(want, st)]
        starts = np.zeros(len(lines) + 1, np.int64)
        np.cumsum(lens, out=starts[1:])
        assert int(starts[-1]) > (1 << 32) + (64 << 20)
        assert np.array_equal(offs, starts)
        assert st[7] != 0 and (np.delete(st, 7) == 0).all()
        h = np.frombuffer(header, np.uint8)
        past = 0
        for i, w in enumerate(want):
            a, b = int(offs[i]), int(offs[i + 1])
            if a == b:
                continue
            assert np.array_equal(buf[a:a + len(header)], h), i
            assert buf[a + len(header):b].tobytes() == w, i
            if a > 1 << 32:  # the boundary: end of the previous record, start of this header
                past += 1
                prev = want[i - 1] if i - 1 != 7 else want[i - 2]
                assert buf[a - len(prev) - 16:a + 16].tobytes() == (header + prev)[-len(prev) - 16:] + header[:16], i
        assert past > 0
    finally:
        dec.close()
