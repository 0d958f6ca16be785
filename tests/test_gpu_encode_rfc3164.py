"""RFC3164 decode + GelfEncoder::encode fused on the device (fg_decode_encode_gelf, fg_split_decode_encode_gelf and the
splitters that use them).  Every record is compared byte for byte with the decode + encode oracle and every status with
fg_decode_batch's.  An RFC3164 Record has no appname, procid or structured data, no severity without <PRI>, and msg is
always Some, possibly "" (rfc3164_decoder.rs:71-82, 106-117), which the GELF text shows.  The year of year-less stamps is
pinned and the system zone database is used, as in test_gpu_z_rfc3164.py.  GPU only."""
import ctypes as C
import re

import numpy as np
import pytest

import vectors as V

pytestmark = pytest.mark.gpu
R3 = 3
YEAR = 2026
INVALID_UTF8 = 76
FLAG_MSG_ARENA = 0x40
# extras override fixed keys, and add the ones an RFC3164 Record leaves out: extras are static items, always written
EXTRAS = [None, {"level": "9", "host": "overridden", "short_message": "x\"y", "application_name": "app", "sd_id": "id\\1"}]
ZONES = ("UTC", "Europe/", "America/", "Asia/", "Etc/", "EST5EDT")
# messages that need escapes or hold multi-byte UTF-8, in line and re-joined into the arena
ESCAPES = [b'<13>Aug  6 11:15:24 h say "hi" \\ there', b"<13>Aug  6 11:15:24 h a\tb\\c", "Aug 6 11:15:24 h café 日本 \U0001F680".encode(),
           "<13>Aug 6 11:15:24 h été  \"x\"\t\\".encode(), b'h: 2020 Aug 6 11:15:24: "q": \\', b"<13>Aug 6 11:15:24 h x\x01y\x1fz"]
_cfgs = {}


def _cfg(oracle, year):
    if year not in _cfgs:
        _cfgs[year] = oracle.Rfc3164Config(year)
    return _cfgs[year]


def _arr(b: bytes) -> np.ndarray:
    return np.frombuffer(b, dtype=np.uint8).copy() if b else np.zeros(0, np.uint8)


def _same_records(buf, offs, ebuf, eo, lines):
    if buf == ebuf and np.array_equal(offs, eo):
        return
    for i in range(len(eo) - 1):
        got, want = buf[offs[i]:offs[i + 1]], ebuf[eo[i]:eo[i + 1]]
        assert got == want, (i, lines[i][:200], got[:300], want[:300])
    raise AssertionError("record extents differ")


def _oracle_gelf(oracle, lines, extra, year=YEAR):
    d, o = oracle.pack(lines)
    return oracle.decode_encode_gelf(R3, d, o, extra or {}, cfg=_cfg(oracle, year), nthreads=16)


def check(dec, oracle, lines, extra=None, year=YEAR):
    """fg_decode_encode_gelf on pre-framed lines against the oracle, statuses against fg_decode_batch.
    Returns (records, statuses, meta of fg_decode_batch)."""
    dec.set_gelf_extra(extra or {})
    d, o = oracle.pack(lines)
    buf, offs, st, _ = dec.decode_encode_gelf(d, o)
    ebuf, eo = _oracle_gelf(oracle, lines, extra, year)
    _same_records(buf, offs, ebuf, eo, lines)
    res = dec.decode(d, o)
    meta = res.meta.copy()
    assert np.array_equal(st, (meta & 0xFF).astype(np.uint8))
    return [buf[offs[i]:offs[i + 1]] for i in range(len(lines))], st, meta


def _frame(stream: bytes, framing: int):
    import pysplit
    return (pysplit.split_nul if framing else pysplit.split_lines)(stream)


def check_split(dec, oracle, native, stream: bytes, framing: int = 0, extra=None, *, prefamed_too: bool = False):
    """fg_split_decode_encode_gelf against the host framing + the oracle; invalid records: status 76 and no bytes."""
    dec.set_gelf_extra(extra or {})
    buf, o, status, line_offs, _ = dec.split_decode_encode_gelf(_arr(stream), framing)
    offs, lines, valid = _frame(stream, framing)
    n = len(lines)
    assert np.array_equal(line_offs, offs)
    assert len(status) == n and len(o) == n + 1 and o[0] == 0
    valid = np.asarray(valid, dtype=bool)
    good = [l for l, v in zip(lines, valid) if v]
    ebuf, eo = _oracle_gelf(oracle, good, extra)
    want_len = np.zeros(n, np.int64)
    want_len[valid] = np.diff(eo)
    if buf != ebuf or not np.array_equal(np.diff(o), want_len):
        k = 0
        for i in range(n):
            want = ebuf[eo[k]:eo[k + 1]] if valid[i] else b""
            assert buf[o[i]:o[i + 1]] == want, (i, lines[i][:200], buf[o[i]:o[i + 1]][:200], want[:200])
            k += int(valid[i])
        raise AssertionError("record extents differ")
    assert np.all(status[~valid] == INVALID_UTF8)
    d, do = oracle.pack(good)
    dec.set_gelf_extra({})
    st_dec = dec.decode(d, do).status.astype(np.uint8) if good else np.zeros(0, np.uint8)
    assert np.array_equal(status[valid], st_dec)
    if prefamed_too:
        dec.set_gelf_extra(extra or {})
        pbuf, po, pst, _ = dec.decode_encode_gelf(d, do)
        assert pbuf == buf and np.array_equal(po, eo) and np.array_equal(pst, status[valid])
    return n


@pytest.fixture(scope="module")
def dec(native):
    d = native.BatchDecoder(native.FMT_RFC3164, max_batch_bytes=96 << 20, max_batch_lines=1 << 20, rfc3164_year=YEAR)
    yield d
    d.close()


@pytest.mark.parametrize("extra", EXTRAS, ids=["plain", "gelf_extra"])
def test_goldens_and_cases(dec, native, oracle, extra):
    lines = [l.encode() for _, _, l, _ in V.RFC3164_GOLDEN] + [l.encode() for l, _ in V.RFC3164_CASES] + ESCAPES
    recs, st, meta = check(dec, oracle, lines, extra)
    ok = st == 0
    n_panic = sum(1 for s in st if s and native.error_string(R3, int(s)) == V.R3_E_PANIC)
    assert n_panic > 0
    assert int((ok & (((meta >> 24) & FLAG_MSG_ARENA) != 0)).sum()) > 0          # re-joined messages read from the arena
    assert sum(1 for l, g in zip(lines, ok) if g and any(z.encode() in l for z in ZONES)) > 0
    good = [r for r, g in zip(recs, ok) if g]
    assert all(r == b"" for r, g in zip(recs, ok) if not g)
    if extra is None:
        assert sum(1 for r in good if b'"level":' not in r) > 0                  # no <PRI>: no level
        assert sum(1 for r in good if b'"level":' in r) > 0
        assert sum(1 for r in good if b'"short_message":""' in r) > 0           # Some(""), not "-"
        assert sum(1 for r in good if b'"host":"unknown"' in r) > 0
        assert not any(k in r for r in good for k in (b'"application_name"', b'"process_id"', b'"sd_id"'))
        assert all(b'"full_message":' in r for r in good)
    else:
        assert all(b'"level":"9"' in r and b'"application_name":"app"' in r and b'"sd_id":"id\\\\1"' in r
                   and b'"host":"overridden"' in r and b'"short_message":"x\\"y"' in r for r in good)
        assert not any(b'"process_id"' in r for r in good)


def test_generated_and_long_lines(dec, native, oracle):
    for seed, n, bad, mean in ((3164, 600_000, 0.02, 0.0), (31, 50_000, 1.0, 0.0), (64, 20_000, 0.005, 600.0)):
        data, offs = native.generate(native.FMT_RFC3164, seed, n, bad_frac=bad, mean_len=mean)
        check(dec, oracle, [bytes(data[offs[i]:offs[i + 1]]) for i in range(n)])
    # lines longer than the encoder's staging tile (at most 4 x 65024 bytes), in line and re-joined into the arena
    long_lines = [b"<13>Aug  6 11:15:24 host " + b'x"\\\ty  ' * 40_000, b"2020 Aug 6 11:15:24 h " + "é\\".encode() * 100_000,
                  b"h: Aug 6 11:15:24: " + b"z: " * 90_000]
    lines = []
    for k, l in enumerate(long_lines):
        lines += [l] + ESCAPES + [b"Aug 6 11:15:24 h m %d" % k] * 300
    recs, st, _ = check(dec, oracle, lines)
    assert all(len(recs[lines.index(l)]) > 260_000 for l in long_lines)
    for extra in EXTRAS:
        check(dec, oracle, lines, extra)


G = b"<13>Aug  6 11:15:24 host tag: m"
LINE_EDGES = [b"", b"\n", b"\n\n", G, G + b"\n", G + b"\r\n", G + b"\r", b"\r\n" + G, G + b"\n\n" + G + b"\n",
              b"\xff\n" + G + b"\n", G + b"\n\xc3", G + b"\n\xc3\n\xa9" + G + b"\n", b"<13>Aug  6 11:15:24 host\r\n",
              b"Aug 6 11:15:24 UTC\n" + G + b"\n\xed\xa0\x80\n" + G, b"a" * 20000 + b"\n" + G + b"\n" + b"b" * 9000,
              b"\n".join(ESCAPES) + b"\n"]
NUL_EDGES = [b"", b"\0", b"\0\0", G, G + b"\0", G + b"\r\n\0", G + b"\0\0" + G + b"\0", b"\xff\0" + G + b"\0", G + b"\0\xc3",
             G + b"\n" + G + b"\0", b"\0".join(ESCAPES)]


@pytest.mark.parametrize("extra", EXTRAS, ids=["plain", "gelf_extra"])
def test_split_framing_edges(dec, native, oracle, extra):
    for stream in LINE_EDGES:
        check_split(dec, oracle, native, stream, 0, extra, prefamed_too=True)
    for stream in NUL_EDGES:
        check_split(dec, oracle, native, stream, 1, extra, prefamed_too=True)


def test_split_generated(dec, native, oracle):
    rng = np.random.default_rng(3164)
    data, offs = native.generate(native.FMT_RFC3164, 77, 200_000, bad_frac=0.02)
    parts = []
    for i in range(200_000):
        l = bytes(data[offs[i]:offs[i + 1]])
        r = rng.random()
        if r < 0.01:
            l = l[: len(l) // 2] + b"\xfe" + l[len(l) // 2:]
        parts.append(l + (b"\r\n" if rng.random() < 0.1 else b"\n"))
    stream = b"".join(parts)
    assert check_split(dec, oracle, native, stream, 0, prefamed_too=True) == 200_000
    assert check_split(dec, oracle, native, stream[:-1].replace(b"\n", b"\0"), 1, prefamed_too=True) == 200_000


def test_split_three_chunks(native, oracle):
    """More than 128 MiB: records straddle both 64 MiB chunk boundaries with a multi-byte character, a truncated
    sequence or a CRLF cut in two; the pre-framed call gives the same records."""
    prefix = b"<13>Aug  6 11:15:24 h "
    line = prefix + b"x" * (63 - len(prefix)) + b"\n"
    B = 64 << 20

    def to(cur, start, parts):
        gap = start - cur
        k = gap // 64 - 1
        parts.append(line * k)
        parts.append(prefix + b"y" * (gap - 64 * k - len(prefix) - 1) + b"\n")
        return start

    d = native.BatchDecoder(native.FMT_RFC3164, max_batch_bytes=160 << 20, max_batch_lines=3 << 20, rfc3164_year=YEAR)
    try:
        for specials in [(("日".encode(), 1), (b"\xe2\x82", 1)), (("\U0001F680".encode(), 3), (b"\r", 1))]:
            parts, cur = [], 0
            for b, (tail, before) in zip((B, 2 * B), specials):
                special = prefix + tail + b"\n"
                cur = to(cur, b - len(prefix) - before, parts)
                parts.append(special)
                cur += len(special)
            parts.append(line * 1000 + prefix + b"end")
            stream = b"".join(parts)
            assert len(stream) > 2 * B
            check_split(d, oracle, native, stream, 0, prefamed_too=True)
    finally:
        d.close()


# 1 MiB / 1024-line context: the arena starts at 64 KiB, the output buffer at 2 x 1 MiB + 200 B per line
ARENA_LINES = [b"<13>Aug  6 11:15:24 h " + b"a  b " * 1000] * 20                    # 80 KB of re-joined messages
OUTPUT_LINES = [b"<13>Aug  6 11:15:24 h m" + b'\\"' * 480] * 1000                  # every byte escaped, twice per record


@pytest.mark.parametrize("lines", [ARENA_LINES, OUTPUT_LINES], ids=["arena", "output-buffer"])
@pytest.mark.parametrize("split", [True, False], ids=["split", "framed"])
def test_regrow(native, oracle, lines, split):
    ebuf, eo = _oracle_gelf(oracle, lines, None)
    assert len(eo) == len(lines) + 1 and np.all(np.diff(eo) > 0)  # every line is a record
    if lines is OUTPUT_LINES:
        assert len(ebuf) > 2 * (1 << 20) + 1024 * 200
    stream = _arr(b"\n".join(lines) + b"\n")
    dd, do = oracle.pack(lines)
    d = native.BatchDecoder(native.FMT_RFC3164, max_batch_bytes=1 << 20, max_batch_lines=1024, rfc3164_year=YEAR)
    try:
        launches = []
        for _ in range(2):
            n0 = d.kernel_launches()
            if split:
                buf, offs, st, _, _ = d.split_decode_encode_gelf(stream, 0)
            else:
                buf, offs, st, _ = d.decode_encode_gelf(dd, do)
            launches.append(d.kernel_launches() - n0)
            assert np.all(st == 0)
            _same_records(buf, offs, ebuf, eo, lines)
        assert launches[0] == 2 * launches[1], launches  # the first call overflowed and redid the batch once
    finally:
        d.close()


_TS = re.compile(rb'"timestamp":[^,}]*')


def test_year_between_fused_calls(dec, oracle):
    lines = [b"<13>Aug  6 11:15:24 h m", b"<13>2020 Aug  6 11:15:24 h m", b"h: Aug 6 11:15:24: m", b"h: 2019 Mar 27 12:09:39: m",
             b"Dec 31 23:59:59 UTC h m", b"2024 Feb 29 11:15:24 h m", b"Aug 6 11:15:24 h", b"nope"]
    yearless = [0, 2, 4, 6]
    try:
        dec.set_rfc3164_year(YEAR)
        a, _, _ = check(dec, oracle, lines, year=YEAR)
        dec.set_rfc3164_year(2024)
        b, _, _ = check(dec, oracle, lines, year=2024)
    finally:
        dec.set_rfc3164_year(YEAR)
    assert [k for k in range(len(lines)) if a[k] != b[k]] == yearless
    assert [_TS.sub(b"", x) for x in a] == [_TS.sub(b"", x) for x in b]


def _raw(d, fmt, stream, split):
    from flowgger_b200.native import FgEncodedOut
    out = FgEncodedOut()
    arr = _arr(stream)
    if split:
        lo = C.POINTER(C.c_int32)()
        rc = d.L.fg_split_decode_encode_gelf(d.ctx, fmt, 0, C.c_void_p(arr.ctypes.data), len(arr), C.byref(out), C.byref(lo))
    else:
        offs = np.array([0, len(arr)], np.int32)
        rc = d.L.fg_decode_encode_gelf(d.ctx, fmt, C.c_void_p(arr.ctypes.data), C.c_void_p(offs.ctypes.data), 1, C.byref(out))
    return rc, d.L.fg_last_error(d.ctx).decode()


def test_other_formats_are_refused(native, oracle):
    d = native.BatchDecoder(native.FMT_RFC3164, max_batch_bytes=1 << 20, max_batch_lines=1 << 12, rfc3164_year=YEAR)
    try:
        for fmt in (native.FMT_LTSV, native.FMT_GELF):
            for split in (True, False):
                rc, err = _raw(d, fmt, G + b"\n", split)
                assert rc == -1 and err == "the fused encoder takes input.format = rfc5424"
        check(d, oracle, [G] + ESCAPES)
        check_split(d, oracle, native, b"\n".join([G] + ESCAPES), 0)
    finally:
        d.close()


def _splitter_records(native, framing):
    data, offs = native.generate(native.FMT_RFC3164, 17, 3000, bad_frac=0.02)
    lines = [bytes(data[offs[i]:offs[i + 1]]) for i in range(3000)]
    lines[5] = lines[5] + b"\r"
    lines[6] = b"<13>Aug  6 11:15:24 h \xff\xfe broken utf8"
    lines[7] = lines[7] + b"\xe2\x82"
    lines[8] = b""
    lines[9] = b"   "
    lines[10] = b"Aug 6 11:15:24 UTC"                                           # FG_E3_PANIC
    lines[11] = b"<13>: Aug  6 11:15:24: m"                                     # empty hostname
    lines[12:12 + len(ESCAPES)] = ESCAPES
    lines[1000] = b"<13>2020 Aug  6 11:15:24 h " + b"y " * (3 << 19)           # longer than the 1 MiB context
    if framing == 2:  # syslen: a record that is not UTF-8 ends the stream
        lines[6] = b"<13>Aug  6 11:15:24 h fine"
        lines[7] = lines[7][:-2]
    return lines[:2000] + [b"x"] * 100_000 + lines[2000:]


def _splitter_text(recs, framing):
    if framing == 2:
        return b"".join(b"%d %s" % (len(r), r) for r in recs)
    d = b"\0" if framing else b"\n"
    return d.join(recs) + d


def _want(oracle, text, recs, framing):
    if framing == 2:
        lines, valid = recs, [True] * len(recs)
    else:
        _, lines, valid = _frame(text, framing)
    good = [l for l, v in zip(lines, valid) if v]
    d, o = oracle.pack(good)
    dbuf, do = oracle.decode_dump(R3, d, o, _cfg(oracle, YEAR), nthreads=16)
    ebuf, eo = oracle.decode_encode_gelf(R3, d, o, {"env": "prod"}, cfg=_cfg(oracle, YEAR), nthreads=16)
    out, errs = [], []
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
            out.append(ebuf[eo[k]:eo[k + 1]])
        k += 1
    if framing == 2:
        errs.append(b"Can't read message's length")  # syslen_splitter.rs:23 at the end of the stream
    return out, errs


@pytest.mark.parametrize("framing", [0, 1, 2], ids=["line", "nul", "syslen"])
def test_splitters_end_to_end(native, oracle, framing):
    recs = _splitter_records(native, framing)
    text = _splitter_text(recs, framing)
    want, errs = _want(oracle, text, recs, framing)
    assert any(e.startswith(V.R3_E_PANIC.encode()) for e in errs)
    d = native.BatchDecoder(native.FMT_RFC3164, max_batch_bytes=1 << 20, max_batch_lines=1 << 12, rfc3164_year=YEAR)
    try:
        records, err = native.splitter_run_gelf(d, text, {"env": "prod"}, max_lines=1 << 16, max_bytes=1 << 20, framing=framing)
        assert records.split(b"\n")[:-1] == want
        assert err.split(b"\n")[:-1] == errs
        _, err2, out = native.splitter_run(d, text, max_lines=1 << 16, max_bytes=1 << 20, framing=framing)
        assert err2 == err and out == b""
    finally:
        d.close()
