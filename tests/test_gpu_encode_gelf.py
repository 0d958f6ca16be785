"""GELF decode + GelfEncoder::encode fused on the device (a GELF relay: fg_decode_encode_gelf, fg_split_decode_encode_gelf
and the splitters that use them).  Every record is compared byte for byte with the decode + encode oracle, given the
wall clock the call stamped its records without "timestamp" with (fg_encoded_gelf_now), and every status with
fg_decode_batch's.  A GELF Record (gelf_decoder.rs:34-125) has no appname, procid or sd_id, level / short_message /
full_message only when the object has them, one "_" + name pair per other member, and strings that are re-escaped from
their unescaped text.  GPU only."""
import json
import re
import time

import numpy as np
import pytest

import vectors as V

pytestmark = pytest.mark.gpu
GELF = 2
INVALID_UTF8 = 76
FLAG_TS_MISSING = 0x01
EXTRAS = [None, {"_x": "extra", "host": "ex-host", "level": "9", "timestamp": "t", "sd_id": "id\\1", "application_name": "app"}]
GELF_ERRORS = ["Invalid GELF input, unable to parse as a JSON object", "Empty GELF input", "Invalid GELF timestamp",
               "GELF host name must be a string", "GELF short message must be a string", "GELF full message must be a string",
               "GELF version must be a string", "Unsupported GELF version", "Invalid severity level",
               "Invalid severity level (too high)", "Invalid value type in structured data", "Missing hostname"]

H = b'"host":"h"'


def obj(*members: bytes) -> bytes:
    return b"{" + b",".join(members) + b"}"


ESCAPES = [b"\\\"", b"\\\\", b"\\/", b"\\b", b"\\f", b"\\n", b"\\r", b"\\t"] + [b"\\u%04x" % c for c in range(0x20)] + \
    [b"\\u0022", b"\\u005c", b"\\u005C", b"\\u00e9", b"\\u00E9", b"\\uffff", b"\\u0800", b"\\ud83d\\ude80", b"\\uD834\\uDD1E"]
ESC_ALL = b"".join(ESCAPES)

EDGES = [
    obj(H), obj(H, b'"timestamp":1'), obj(H, b'"timestamp":-5'), obj(H, b'"timestamp":-0.0'), obj(H, b'"timestamp":1e21'),
    obj(H, b'"timestamp":5e-324'), obj(H, b'"timestamp":2.2250738585072011e-308'), obj(H, b'"timestamp":18446744073709551615'),
    obj(H, b'"timestamp":-9223372036854775808'), obj(H, b'"timestamp":1385053862.3072'), obj(H, b'"timestamp":0'),
    obj(b'"host":""'), obj(H, b'"short_message":""'), obj(H, b'"short_message":"m"'), obj(H, b'"full_message":"f"'),
    obj(H, b'"full_message":""'), obj(H, b'"level":0'), obj(H, b'"level":7'), obj(H, b'"version":"1.0"'),
    obj(H, b'"version":"1.1"', b'"short_message":"s"', b'"full_message":"f"', b'"level":3', b'"timestamp":12.5'),
    # escapes in host, both messages, pair names and values
    obj(b'"host":"' + ESC_ALL + b'"', b'"short_message":"' + ESC_ALL + b'"', b'"full_message":"' + ESC_ALL + b'"'),
    obj(H, b'"v":"' + ESC_ALL + b'"', b'"' + ESC_ALL + b'":1'),
    *[obj(H, b'"k' + e + b'":"a' + e + b'b"', b'"short_message":"' + e + b'"') for e in ESCAPES],
    obj(H, b'"a\\u0062":1', b'"ab":2'), obj(H, b'"ab":2', b'"a\\u0062":1'), obj(H, b'"\\u005fa":1', b'"a":2'),
    obj(H, b'"a":2', b'"\\u005fa":1'), obj(H, b'"_\\u0061":1', b'"a":3'), obj(H, b'"\\u005f":1', b'"":2'),
    obj(H, b'"\\u0068ost":"esc-host"'), obj(H, b'"x\\u0000y":1', b'"x":2', b'"x\\u0000":3'),
    # key collisions and duplicates
    obj(H, b'"a":1', b'"_a":2'), obj(H, b'"_a":2', b'"a":1'), obj(H, b'"A":1', b'"_A":2'), obj(H, b'"_A":2', b'"A":1'),
    obj(H, b'"a":1', b'"a":2', b'"a":3'), obj(H, b'"host":"h2"'), obj(b'"host":"h1"', b'"host":"h2"', b'"level":1', b'"level":2'),
    obj(H, b'"_":1', b'"":2'), obj(H, b'"_version":1', b'"_host":2', b'"_timestamp":3'), obj(H, b'"_x":1', b'"x":2'),
    # values
    obj(H, b'"t":true', b'"f":false', b'"n":null', b'"i":-9223372036854775808', b'"u":18446744073709551615'),
    obj(H, b'"f1":-0.0', b'"f2":1e21', b'"f3":1e20', b'"f4":1e-7', b'"f5":5e-324', b'"f6":1.7976931348623157e308',
        b'"f7":0.1', b'"f8":123456789012345678901234567890', b'"f9":-1', b'"g":0', b'"h":-0'),
    # whitespace and UTF-8
    b' { "host" : "h" , "x" : [ ] } ', b'{"host":"h","x":{}}', "{\"host\":\"日本\",\"näme\":\"ü\",\"место\":\"ʼ\"}".encode(),
    obj(H, b'"short_message":"a\xc3\xa9\xf0\x9f\x9a\x80"'),
]

# lines with a raw LF go through the decoder's newline retry (gelf_decoder.rs:44-46); `\` + LF becomes `\\n`
RETRY = [b'{"host":"h","short_message":"a\nb"}', b'{"host":"h\n","full_message":"x\\\ny","k\\\n":"v\\\n\\u00e9"}',
         b'{"host":"h","m":"\n\n","n\\u0041\n":"\\\\\n"}']


def _many(k: int, seed: int) -> bytes:
    """an object of k members: names that repeat, collide ("a" / "_a"), hold escapes, and sort around the fixed keys"""
    rng = np.random.default_rng(seed)
    parts = [H]
    for j in range(k):
        nm = [b"a%02d" % (j % 13), b"_a%02d" % (j % 11), b"l\\u0065vel%d" % (j % 5), b"zz%d" % j, b"hosu", b"_\\u0078"][j % 6]
        val = [b'"v\\"%d\\\\"' % j, b"%d" % (j * 7919), b"true", b"null", b'"\\u00e9%d"' % j, b"-%d.5" % j][int(rng.integers(6))]
        parts.append(b'"' + nm + b'":' + val)
    return obj(*parts, b'"short_message":"' + b"\\n" * k + b'"')


LONG = [_many(k, k) for k in (23, 24, 25, 26, 40, 60, 200)]
# segments past the 56-segment windows, with an escaped segment on each boundary
WINDOWS = [obj(H, *[b'"p%03d":"%s"' % (j, b"\\u00e9" if j % 3 else b"x") for j in range(n)]) for n in (17, 18, 19, 36, 37, 38, 80)]


def _arr(b: bytes) -> np.ndarray:
    return np.frombuffer(b, dtype=np.uint8).copy() if b else np.zeros(0, np.uint8)


def _same_records(buf, offs, ebuf, eo, lines):
    if buf == ebuf and np.array_equal(offs, eo):
        return
    for i in range(len(eo) - 1):
        got, want = buf[offs[i]:offs[i + 1]], ebuf[eo[i]:eo[i + 1]]
        assert got == want, (i, lines[i][:300], got[:500], want[:500])
    raise AssertionError("record extents differ")


def oracle_at(oracle, dec, d, o, extra, now):
    """The oracle's decode + encode of the lines with `now` as Record.ts of every record without "timestamp".  The
    oracle leaves that Record.ts at 0.0 (the reference reads the wall clock there); the lines without one are the rows
    fg_decode_batch flags FG_FLAG_TS_MISSING, and their "timestamp":0.0 becomes serde_json's text of `now`."""
    ebuf, eo = oracle.decode_encode_gelf(GELF, d, o, extra or {}, nthreads=16)
    meta = dec.decode(d, o).meta.astype(np.int64)
    missing = np.flatnonzero(((meta & 0xFF) == 0) & (((meta >> 24) & FLAG_TS_MISSING) != 0))
    if len(missing) == 0:
        return ebuf, eo
    zero, at = b',"timestamp":0.0,', b',"timestamp":' + oracle.format_f64(now).encode() + b','
    recs = [ebuf[eo[i]:eo[i + 1]] for i in range(len(eo) - 1)]
    for i in missing:
        assert recs[i].count(zero) == (0 if extra and "timestamp" in extra else 1), recs[i][:300]
        recs[i] = recs[i].replace(zero, at)
    offs = np.zeros(len(recs) + 1, np.int64)
    np.cumsum([len(r) for r in recs], out=offs[1:])
    return b"".join(recs), offs


def check(dec, oracle, lines, extra=None):
    """fg_decode_encode_gelf on pre-framed lines against the oracle with the call's clock; statuses against
    fg_decode_batch.  Returns (records, statuses, now)."""
    dec.set_gelf_extra(extra or {})
    d, o = oracle.pack(lines)
    t0 = time.time()
    buf, offs, st, _ = dec.decode_encode_gelf(d, o)
    t1 = time.time()
    now = dec.gelf_now()
    assert t0 - 1e-3 <= now <= t1 + 1e-3
    ebuf, eo = oracle_at(oracle, dec, d, o, extra, now)
    _same_records(buf, offs, ebuf, eo, lines)
    res = dec.decode(d, o)
    assert np.array_equal(st, (res.meta & 0xFF).astype(np.uint8))
    return [buf[offs[i]:offs[i + 1]] for i in range(len(lines))], st, now


@pytest.fixture(scope="module")
def dec(native):
    d = native.BatchDecoder(GELF, max_batch_bytes=96 << 20, max_batch_lines=1 << 20)
    yield d
    d.close()


@pytest.mark.parametrize("extra", EXTRAS, ids=["plain", "gelf_extra"])
def test_goldens_cases_and_errors(dec, native, oracle, extra):
    lines = [V.G3_LINE.encode()] + [l.encode() if isinstance(l, str) else l for l, _ in V.GELF_CASES] + [obj(H, b'"level":8')]
    recs, st, _ = check(dec, oracle, lines, extra)
    errs = {native.error_string(GELF, int(s)) for s in st if s}
    assert set(GELF_ERRORS) <= errs, set(GELF_ERRORS) - errs
    assert all(r == b"" for r, s in zip(recs, st) if s)
    assert st[0] == 0 and len(recs[0]) > 0


@pytest.mark.parametrize("extra", EXTRAS, ids=["plain", "gelf_extra"])
def test_edges(dec, oracle, extra):
    lines = EDGES + RETRY + LONG + WINDOWS
    recs, st, now = check(dec, oracle, lines, extra)
    bad = {b' { "host" : "h" , "x" : [ ] } ', b'{"host":"h","x":{}}'}  # a container as a member value
    assert all((s != 0) == (l in bad) for l, s in zip(lines, st)), [(l, s) for l, s in zip(lines, st) if s]
    r = dict(zip(lines, recs))
    for rec in recs:
        if rec:
            json.loads(rec, strict=False)  # serde_json text is JSON (control bytes other than \\b \\f \\n \\r \\t stay raw)
    if extra is None:
        assert b'"version":"1.1"' in r[obj(H, b'"version":"1.0"')]
        assert b'"short_message":"-"' in r[obj(H)] and b'"short_message":""' in r[obj(H, b'"short_message":""')]
        assert b'"full_message"' not in r[obj(H)] and b'"full_message":""' in r[obj(H, b'"full_message":""')]
        assert b'"level"' not in r[obj(H)] and b'"level":0' in r[obj(H, b'"level":0')]
        assert b'"host":"unknown"' in r[obj(b'"host":""')]
        assert r[obj(H, b'"a":1', b'"_a":2')].count(b'"_a":') == 1 and b'"_a":1' in r[obj(H, b'"a":1', b'"_a":2')]
        assert b'"_A":2' in r[obj(H, b'"A":1', b'"_A":2')]
        assert b'"_k/":"a/b"' in r[obj(H, b'"k\\/":"a\\/b"', b'"short_message":"\\/"')]
        assert b'"_n":null' in r[EDGES[-6]] and b'"_u":18446744073709551615' in r[EDGES[-6]]
        assert json.loads(r[obj(H)])["timestamp"] == pytest.approx(now, abs=1e-5)
        assert b'"short_message":"a\\nb"' in r[RETRY[0]]
    else:
        assert all(b'"timestamp":"t"' in x and b'"host":"ex-host"' in x and b'"sd_id":"id\\\\1"' in x for x in recs if x)


def test_missing_timestamps_share_the_call_clock(native, oracle):
    d = native.BatchDecoder(GELF, max_batch_bytes=1 << 20, max_batch_lines=1 << 12)
    try:
        lines = [obj(H, b'"i":%d' % i) if i % 3 else obj(H, b'"timestamp":%d' % i) for i in range(3000)]
        recs, st, now = check(d, oracle, lines)
        stamps = {json.loads(r)["timestamp"] for i, r in enumerate(recs) if i % 3}
        assert len(stamps) == 1 and stamps.pop() == pytest.approx(now, abs=1e-5)
        _, _, now2 = check(d, oracle, lines)
        assert now2 >= now
    finally:
        d.close()


def test_generated_prefamed_and_split(native, oracle):
    """200 k bench-shaped lines (escape-rich full_message): against the oracle, and the split calls (LF framing for lines
    without a raw LF, NUL framing for all) against the pre-framed one"""
    n = 200_000
    data, offs = native.generate(GELF, 0x6E1F, n, bad_frac=0.02)
    lines = [bytes(data[offs[i]:offs[i + 1]]) for i in range(n)]
    dec = native.BatchDecoder(GELF, max_batch_bytes=192 << 20, max_batch_lines=1 << 20)
    rng = np.random.default_rng(7)
    try:
        for extra in EXTRAS:
            recs, st, _ = check(dec, oracle, lines, extra)
            assert (st == 0).sum() > 190_000
            for framing, sel in ((0, [l for l in lines if b"\n" not in l]), (1, [l for l in lines if b"\0" not in l])):
                term = b"\0" if framing else b"\n"
                parts = [l + (b"\r\n" if (not framing and rng.random() < 0.1) else term) for l in sel]
                sbuf, so, sst, sl, _ = dec.split_decode_encode_gelf(_arr(b"".join(parts)), framing)
                snow = dec.gelf_now()
                d, o = oracle.pack(sel)
                ebuf, eo = oracle_at(oracle, dec, d, o, extra, snow)
                _same_records(sbuf, so, ebuf, eo, sel)
                res = dec.decode(d, o)
                assert np.array_equal(sst, (res.meta & 0xFF).astype(np.uint8))
    finally:
        dec.close()


def _frame(stream: bytes, framing: int):
    import pysplit
    return (pysplit.split_nul if framing else pysplit.split_lines)(stream)


LINE_EDGES = [b"", b"\n", obj(H), obj(H) + b"\r\n", b"\xff\n" + obj(H) + b"\n", obj(H) + b"\n\xc3",
              b"\n".join(l for l in EDGES + LONG + WINDOWS) + b"\n"]
NUL_EDGES = [b"", b"\0", obj(H) + b"\0", b"\0".join(EDGES + RETRY + LONG) + b"\0", b"\xff\0" + RETRY[1] + b"\0" + RETRY[0]]


@pytest.mark.parametrize("extra", EXTRAS, ids=["plain", "gelf_extra"])
def test_split_framing_edges(dec, oracle, extra):
    dec.set_gelf_extra(extra or {})
    for framing, streams in ((0, LINE_EDGES), (1, NUL_EDGES)):
        for stream in streams:
            buf, o, status, line_offs, _ = dec.split_decode_encode_gelf(_arr(stream), framing)
            now = dec.gelf_now()
            offs, lines, valid = _frame(stream, framing)
            valid = np.asarray(valid, dtype=bool)
            assert np.array_equal(line_offs, offs) and len(status) == len(lines)
            good = [l for l, v in zip(lines, valid) if v]
            d, do = oracle.pack(good)
            ebuf, eo = oracle_at(oracle, dec, d, do, extra, now)
            want_len = np.zeros(len(lines), np.int64)
            want_len[valid] = np.diff(eo)
            assert buf == ebuf and np.array_equal(np.diff(o), want_len), stream[:200]
            assert np.all(status[~valid] == INVALID_UTF8)


# 1 MiB / 1024-line context: the side table and the output buffer both start too small
PAIR_LINES = [obj(H, *[b'"k%d":"v"' % j for j in range(60)]) for _ in range(1000)]
# 1e20 is written 100000000000000000000.0 and a raw LF (newline retry) \n: twice the input, rows well inside the side table
OUTPUT_LINES = [obj(H, *[b'"a%02d":1e20' % j for j in range(40)], b'"short_message":"' + b"\n" * 560 + b'"')] * 1000


@pytest.mark.parametrize("lines", [PAIR_LINES, OUTPUT_LINES], ids=["side-table", "output-buffer"])
@pytest.mark.parametrize("split", [True, False], ids=["split", "framed"])
def test_regrow(native, oracle, lines, split):
    framing = 1 if lines is OUTPUT_LINES else 0  # records with a raw LF are NUL-framed
    dl = b"\0" if framing else b"\n"
    stream = _arr(dl.join(lines) + dl)
    dd, do = oracle.pack(lines)
    d = native.BatchDecoder(GELF, max_batch_bytes=1 << 20, max_batch_lines=1024)
    try:
        launches = []
        for _ in range(2):
            n0 = d.kernel_launches()
            if split:
                buf, offs, st, _, _ = d.split_decode_encode_gelf(stream, framing)
            else:
                buf, offs, st, _ = d.decode_encode_gelf(dd, do)
            launches.append(d.kernel_launches() - n0)
            assert np.all(st == 0)
            ebuf, eo = oracle_at(oracle, d, dd, do, {}, d.gelf_now())
            _same_records(buf, offs, ebuf, eo, lines)
        assert launches[0] == 2 * launches[1], launches
        check(d, oracle, EDGES + LONG)
    finally:
        d.close()


def _raw_fused(d, fmt, stream: bytes, split: bool):
    import ctypes as C
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


def test_refusals(native, oracle):
    """GELF input on an RFC5424 context is refused with the unchanged text; gelf_now fails after a non-GELF call and
    ltsv_stops after a GELF call; the contexts keep working"""
    refused = "the fused encoder takes input.format = rfc5424"
    g = native.BatchDecoder(GELF, max_batch_bytes=1 << 20, max_batch_lines=1 << 12)
    r5 = native.BatchDecoder(native.FMT_RFC5424, max_batch_bytes=1 << 20, max_batch_lines=1 << 12)
    try:
        for split in (True, False):
            assert _raw_fused(r5, GELF, obj(H) + b"\n", split) == (-1, refused)
            with pytest.raises(RuntimeError, match="fg_encoded_gelf_now"):
                r5.gelf_now()
        dd, do = oracle.pack([V.G1_LINE.encode(), V.G2_LINE.encode()])
        r5.decode_encode_gelf(dd, do)
        with pytest.raises(RuntimeError, match="fg_encoded_gelf_now"):
            r5.gelf_now()
        check(g, oracle, EDGES)
        with pytest.raises(RuntimeError, match="fg_encoded_ltsv_stops"):
            g.ltsv_stops()
        assert _raw_fused(g, native.FMT_RFC5424, b"x\n", True)[0] == 0
        with pytest.raises(RuntimeError, match="fg_encoded_gelf_now"):
            g.gelf_now()
        check(g, oracle, EDGES)
    finally:
        g.close()
        r5.close()


_TS = re.compile(rb'([,{])"timestamp":(-?[0-9][0-9.e+-]*)([,}])')


def _splitter_records(native, framing):
    data, offs = native.generate(GELF, 17, 3000, bad_frac=0.02)
    lines = [bytes(data[offs[i]:offs[i + 1]]) for i in range(3000)]
    lines = [l for l in lines if b"\n" not in l and b"\0" not in l]
    lines[5] = lines[5] + b"\r"
    lines[6] = b'{"host":"h","x":"\xff\xfe"}'
    lines[8] = b""
    lines[9] = b"   "
    lines[12:12 + len(EDGES)] = EDGES
    lines[1000] = obj(H, b'"short_message":"' + b"y " * (3 << 19) + b'"')  # longer than the 1 MiB context
    if framing == 2:
        lines[6] = obj(H, b'"x":"fine"')
    return lines[:2000] + [b"x"] * 20_000 + lines[2000:]


@pytest.mark.parametrize("framing", [0, 1, 2], ids=["line", "nul", "syslen"])
def test_splitters_end_to_end(native, oracle, framing):
    """records against the oracle's encoder (a record without "timestamp" compared through the clock it carries, which
    lies inside the run); stderr identical to the non-fused splitter on the same input"""
    recs = _splitter_records(native, framing)
    if framing == 2:
        text = b"".join(b"%d %s" % (len(r), r) for r in recs)
        lines, valid = recs, [True] * len(recs)
    else:
        dl = b"\0" if framing else b"\n"
        text = dl.join(recs) + dl
        _, lines, valid = _frame(text, framing)
    good = [l for l, v in zip(lines, valid) if v]
    d, o = oracle.pack(good)
    ebuf, eo = oracle.decode_encode_gelf(GELF, d, o, {"env": "prod"}, nthreads=16)  # Record.ts 0.0 without "timestamp"
    want = [ebuf[eo[k]:eo[k + 1]] for k in range(len(good)) if eo[k + 1] > eo[k]]
    dec = native.BatchDecoder(GELF, max_batch_bytes=1 << 20, max_batch_lines=1 << 12)
    try:
        t0 = time.time()
        records, err = native.splitter_run_gelf(dec, text, {"env": "prod"}, max_lines=1 << 16, max_bytes=1 << 20, framing=framing)
        t1 = time.time()
        got = records.split(b"\n")[:-1]
        assert len(got) == len(want)
        zero = b'"timestamp":0.0'
        for g, w in zip(got, want):
            if g == w:
                continue
            assert zero in w, (g[:300], w[:300])
            m = _TS.search(g)
            assert m and t0 - 1e-3 <= float(m.group(2)) <= t1 + 1e-3
            assert _TS.sub(rb'\1"timestamp":0.0\3', g, count=1) == w
        _, err2, _ = native.splitter_run(dec, text, max_lines=1 << 16, max_bytes=1 << 20, framing=framing)
        assert err == err2 and err.count(b"\n") > 20_000
    finally:
        dec.close()
