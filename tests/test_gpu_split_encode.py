"""Framing + UTF-8 check + RFC5424 decode + GelfEncoder::encode of a raw stream in one device call
(fg_split_decode_encode_gelf), and the batching splitters that use it.  Expected bytes come from the CPU restatement of
the framing (oracle/pysplit.py) and the decode + encode oracle: a valid record gives the oracle's JSON, an invalid one
status 76 ("Invalid UTF-8 input") and an empty record.  GPU only."""
import ctypes as C

import numpy as np
import pytest

import vectors as V

pytestmark = pytest.mark.gpu
R5 = 0
INVALID_UTF8 = 76
EXTRAS = [None, {"env": "prod", "host": "overridden", "a\"b": "c\\d\n"}]


def _arr(stream: bytes) -> np.ndarray:
    return np.frombuffer(stream, dtype=np.uint8) if stream else np.zeros(0, np.uint8)


def _frame(stream: bytes, framing: int):
    import pysplit
    return (pysplit.split_nul if framing else pysplit.split_lines)(stream)


def check(dec, oracle, native, stream: bytes, framing: int = 0, extra=None, *, prefamed_too: bool = False):
    """The device call against the oracle; returns the number of records."""
    dec.set_gelf_extra(extra or {})
    buf, o, status, line_offs, _ = dec.split_decode_encode_gelf(_arr(stream), framing)
    offs, lines, valid = _frame(stream, framing)
    n = len(lines)
    assert np.array_equal(line_offs, offs), (line_offs[:10], offs[:10])
    assert len(status) == n and len(o) == n + 1 and o[0] == 0
    valid = np.asarray(valid, dtype=bool)
    good = [l for l, v in zip(lines, valid) if v]
    d, do = oracle.pack(good)
    ebuf, eo = oracle.decode_encode_gelf(R5, d, do, extra or {}, nthreads=16)
    # an invalid record has no bytes, so the concatenation is the oracle's over the valid records
    want_len = np.zeros(n, np.int64)
    want_len[valid] = np.diff(eo)
    if buf != ebuf or not np.array_equal(np.diff(o), want_len):
        k = 0
        for i in range(n):
            got = buf[o[i]:o[i + 1]]
            want = ebuf[eo[k]:eo[k + 1]] if valid[i] else b""
            assert got == want, (i, lines[i][:200], got[:200], want[:200])
            k += int(valid[i])
        raise AssertionError("record extents differ")
    assert np.all(status[~valid] == INVALID_UTF8)
    # the decoder's status on the valid records: its error text is the oracle's
    dbuf, dbo = oracle.decode_dump(R5, d, do, nthreads=16)
    rejected = np.frombuffer(dbuf, dtype=np.uint8)[dbo[:-1]] == ord("E") if len(good) else np.zeros(0, bool)
    st = status[valid]
    assert np.array_equal(st != 0, rejected)
    for k in np.flatnonzero(rejected)[:2000]:
        dump = dbuf[dbo[k]:dbo[k + 1]]
        assert native.error_string(R5, int(st[k])).encode() == dump[2:dump.index(b";out=")]
    if prefamed_too:
        # the same valid lines framed on the host and handed to fg_decode_encode_gelf
        pbuf, po, pst, _ = dec.decode_encode_gelf(d, do)
        assert pbuf == buf and np.array_equal(po, eo) and np.array_equal(pst, st)
    return n


@pytest.fixture(scope="module")
def dec(native):
    d = native.BatchDecoder(native.FMT_RFC5424, max_batch_bytes=64 << 20, max_batch_lines=1 << 18)
    yield d
    d.close()


G = V.G1_LINE.encode()
LINE_EDGES = [b"", b"\n", b"\n\n", G, G + b"\n", G + b"\r\n", G + b"\r", G + b"\r\r\n", b"\r\n" + G, G + b"\n" + G,
              G + b"\n\n" + G + b"\n", b"\xff\n" + G + b"\n", G + b"\n\xc3", G + b"\n\xc3\n\xa9" + G + b"\n",
              "<13>1 2015-08-05T15:53:45Z h a p m - café 日本\U0001F680\n".encode(),
              b"<13>1 x \xed\xa0\x80\n" + G + b"\n\xf4\x90\x80\x80\n\xe0\x80\x80\n\xc0\xaf\n" + G,
              b"a" * 20000 + b"\n" + G + b"\n" + b"b" * 9000,
              G + b"\n" + ("<13>1 2015-08-05T15:53:45Z h a p m - " + "z" * 20000).encode() + b"\r\n" + V.G2_LINE.encode()]
NUL_EDGES = [b"", b"\0", b"\0\0", G, G + b"\0", G + b"\r\n\0", G + b"\0" + G, G + b"\0\0" + G + b"\0", b"\xff\0" + G + b"\0",
             G + b"\0\xc3", G + b"\n" + G + b"\0", b"a" * 20000 + b"\0" + G + b"\0" + b"b" * 9000]


@pytest.mark.parametrize("extra", EXTRAS, ids=["plain", "gelf_extra"])
def test_line_framing_edge_cases(dec, oracle, native, extra):
    for stream in LINE_EDGES:
        check(dec, oracle, native, stream, 0, extra)


@pytest.mark.parametrize("extra", EXTRAS, ids=["plain", "gelf_extra"])
def test_nul_framing_edge_cases(dec, oracle, native, extra):
    for stream in NUL_EDGES:
        check(dec, oracle, native, stream, 1, extra)


def _generated_lines(native, seed, n, bad_frac):
    data, offs = native.generate(native.FMT_RFC5424, seed, n, bad_frac=bad_frac)
    return [bytes(data[offs[i]:offs[i + 1]]) for i in range(n)]


def test_generated_stream(dec, oracle, native):
    """200 k lines with 1 % invalid bytes, 1 % truncated sequences at the end of a line, 10 % CRLF and the generator's
    decoder rejects; the valid lines also match fg_decode_encode_gelf over the same lines framed on the host."""
    rng = np.random.default_rng(5424)
    parts = []
    for l in _generated_lines(native, 31, 200_000, 0.02):
        r = rng.random()
        if r < 0.01:
            l = l[: len(l) // 2] + b"\xfe" + l[len(l) // 2:]
        elif r < 0.02:
            l = l + b"\xe2\x82"
        parts.append(l + (b"\r\n" if rng.random() < 0.1 else b"\n"))
    stream = b"".join(parts)
    for extra in EXTRAS:
        assert check(dec, oracle, native, stream, 0, extra, prefamed_too=True) == 200_000
    assert check(dec, oracle, native, stream[:-1], 0) == 200_000  # unterminated last line


def test_generated_nul_stream(dec, oracle, native):
    lines = _generated_lines(native, 23, 100_000, 0.01)
    lines[7] = lines[7] + b"\r\n"  # ordinary bytes under NUL framing
    lines[8] = b"\xff" + lines[8]
    assert check(dec, oracle, native, b"\0".join(lines) + b"\0", 1, prefamed_too=False) == 100_000


def test_three_chunk_stream(native, oracle):
    """More than 128 MiB: the call pipelines 64 MiB chunks.  At both chunk boundaries a record straddles the boundary
    with a multi-byte character, a truncated or invalid sequence, or a CRLF split in two."""
    prefix = b"<13>1 2015-08-05T15:53:45Z h a p m - "
    line = prefix + b"x" * (63 - len(prefix)) + b"\n"  # 64 bytes
    assert len(line) == 64
    B = 64 << 20

    def to(cur, start, parts):
        # whole lines up to `start`, the last one stretched to land exactly on it
        gap = start - cur
        k = gap // 64 - 1
        parts.append(line * k)
        parts.append(prefix + b"y" * (gap - 64 * k - len(prefix) - 1) + b"\n")
        return start

    dec = native.BatchDecoder(native.FMT_RFC5424, max_batch_bytes=160 << 20, max_batch_lines=3 << 20)
    try:
        for specials in [((("日".encode(), 1)), (b"\xe2\x82", 1)), (("\U0001F680".encode(), 3), (b"\r", 1)),
                         ((b"\xc3", 0), ("é".encode(), 1))]:
            parts, cur = [], 0
            for b, (tail, before) in zip((B, 2 * B), specials):
                special = prefix + tail + b"\n"
                cur = to(cur, b - len(prefix) - before, parts)
                parts.append(special)
                cur += len(special)
            parts.append(line * 1000 + prefix + b"end")  # a third chunk, unterminated last line
            stream = b"".join(parts)
            assert len(stream) > 2 * B
            check(dec, oracle, native, stream, 0)
    finally:
        dec.close()


# Messages of backslashes and tabs, no structured data: each byte is escaped in short_message and in full_message, so
# the records are about four times the input, more than the first output buffer of a 1 MiB / 1024-line context
# (2 x 1 MiB + 200 B per line), while no side table is used
TINY_LINES = [b"<13>1 2015-08-05T15:53:45Z h a p m - m" + b"\\\t" * 480 + b"m"] * 1000
# 400 one-pair elements per line: the RFC5424 side tables overflow their first sizes, the output buffer does not
WIDE_SD_LINES = [(V.H + "".join('[i k="v"]' for _ in range(400)) + " m").encode()] * 900


@pytest.mark.parametrize("lines,max_bytes,max_lines", [(TINY_LINES, 1 << 20, 1024), (WIDE_SD_LINES, 8 << 20, 900)],
                         ids=["output-buffer", "side-table"])
def test_regrow(native, oracle, lines, max_bytes, max_lines):
    stream = b"\n".join(lines) + b"\n"
    assert len(stream) <= max_bytes
    if lines is TINY_LINES:
        d, o = oracle.pack(lines)
        assert len(oracle.decode_encode_gelf(R5, d, o)[0]) > 2 * max_bytes + max_lines * 200
    dec = native.BatchDecoder(native.FMT_RFC5424, max_batch_bytes=max_bytes, max_batch_lines=max_lines)
    try:
        launches = []
        for _ in range(2):
            n0 = dec.kernel_launches()
            check(dec, oracle, native, stream, 0)
            launches.append(dec.kernel_launches() - n0)
        assert launches[0] == 2 * launches[1], launches  # the first call overflowed and redid the batch once
    finally:
        dec.close()


def _raw_call(dec, fmt, framing, stream):
    """fg_split_decode_encode_gelf with any format: (return code, fg_last_error)"""
    from flowgger_b200.native import FgEncodedOut
    out = FgEncodedOut()
    lo = C.POINTER(C.c_int32)()
    rc = dec.L.fg_split_decode_encode_gelf(dec.ctx, fmt, framing, C.c_void_p(stream.ctypes.data), len(stream), C.byref(out), C.byref(lo))
    return rc, dec.L.fg_last_error(dec.ctx).decode()


def test_error_returns_leave_the_context_usable(native, oracle):
    dec = native.BatchDecoder(native.FMT_RFC5424, max_batch_bytes=1 << 20, max_batch_lines=1 << 12)
    try:
        ok = _arr(b"\n".join(_generated_lines(native, 9, 2000, 0.02)) + b"\n")
        rc, err = _raw_call(dec, native.FMT_LTSV, 0, ok)
        assert rc == -1 and err == "the fused encoder takes input.format = rfc5424"
        rc, err = _raw_call(dec, native.FMT_RFC5424, 2, ok)
        assert rc == -1 and err == "unknown framing"
        rc, err = _raw_call(dec, native.FMT_RFC5424, 0, np.full((1 << 20) + 1, ord("\n"), np.uint8))
        assert rc == -3 and err == "stream has more bytes than max_batch_bytes"
        rc, err = _raw_call(dec, native.FMT_RFC5424, 1, np.zeros(10_000, np.uint8))  # 10 000 empty NUL records
        assert rc == -3 and err == "stream has more lines than max_batch_lines"
        rc, err = _raw_call(dec, native.FMT_RFC5424, 0, np.tile(np.frombuffer(b"x\n", np.uint8), 100_000))
        assert rc == -3 and err == "stream has more lines than max_batch_lines"
        check(dec, oracle, native, bytes(ok), 0)
        check(dec, oracle, native, bytes(ok).replace(b"\n", b"\0"), 1)
    finally:
        dec.close()


def _splitter_text(native, framing):
    d = b"\0" if framing else b"\n"
    lines = _generated_lines(native, 17, 3000, 0.02)
    lines[5] = lines[5] + b"\r"                       # CRLF under line framing, ordinary bytes under NUL
    lines[6] = b"<13>1 \xff\xfe broken utf8"          # "Invalid UTF-8 input"
    lines[7] = lines[7][:-1] + b"\xe2\x82"            # truncated sequence at the end
    lines[8] = b""                                    # blank records: reported by the line splitter only
    lines[9] = b"   "
    lines[1000] = b"<13>1 " + V.TS.encode() + b" h a p m - " + b"y" * (3 << 20)  # longer than the 1 MiB context
    recs = lines[:2000] + [b"x"] * 100_000 + lines[2000:]  # 100 k two-byte records: far more than the context's 4096 lines
    return d.join(recs) + d


def _want(oracle, text, framing, gelf):
    offs, lines, valid = _frame(text, framing)
    good = [l for l, v in zip(lines, valid) if v]
    d, o = oracle.pack(good)
    dbuf, do = oracle.decode_dump(R5, d, o, nthreads=16)
    ebuf, eo = oracle.decode_encode_gelf(R5, d, o, {"env": "prod"}, nthreads=16) if gelf else (None, None)
    recs, errs = [], []
    k = 0
    for l, v in zip(lines, valid):
        if not v:
            errs.append(b"Invalid UTF-8 input")
            continue
        dump = dbuf[do[k]:do[k + 1]]
        if dump.startswith(b"E:"):
            t = l.decode().strip().encode()
            if not (framing == 1 and not t):  # nul_splitter.rs:41-45
                errs.append(dump[2:dump.index(b";out=")] + b": [" + t + b"]")
        else:
            recs.append(ebuf[eo[k]:eo[k + 1]] if gelf else dump[:dump.rindex(b";out=")] + b";out=0")
        k += 1
    return recs, errs


@pytest.mark.parametrize("framing", [0, 1], ids=["line", "nul"])
def test_fused_splitter_end_to_end(native, oracle, framing):
    text = _splitter_text(native, framing)
    dec = native.BatchDecoder(native.FMT_RFC5424, max_batch_bytes=1 << 20, max_batch_lines=1 << 12)
    try:
        records, err = native.splitter_run_gelf(dec, text, {"env": "prod"}, max_lines=1 << 16, max_bytes=1 << 20, framing=framing)
    finally:
        dec.close()
    recs, errs = _want(oracle, text, framing, True)
    assert records.split(b"\n")[:-1] == recs
    assert err.split(b"\n")[:-1] == errs


@pytest.mark.parametrize("framing", [0, 1], ids=["line", "nul"])
def test_splitter_block_capacity(native, oracle, framing):
    """The same stream through the splitters without the fused encoder (records materialised on the host)."""
    text = _splitter_text(native, framing)
    dec = native.BatchDecoder(native.FMT_RFC5424, max_batch_bytes=1 << 20, max_batch_lines=1 << 12)
    try:
        records, err, out = native.splitter_run(dec, text, max_lines=1 << 16, max_bytes=1 << 20, framing=framing)
    finally:
        dec.close()
    recs, errs = _want(oracle, text, framing, False)
    assert records.split(b"\n")[:-1] == recs
    assert err.split(b"\n")[:-1] == errs
    assert out == b""
