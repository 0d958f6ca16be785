"""LTSV decode + GelfEncoder::encode fused on the device (fg_decode_encode_gelf, fg_split_decode_encode_gelf and the
splitters that use them).  Every record is compared byte for byte with the decode + encode oracle, every status with
fg_decode_batch's, and every "Missing value" stop (fg_encoded_ltsv_stops) with what the non-fused path prints.  An LTSV
Record (ltsv_decoder.rs:87-221) has no appname, procid or sd_id, no severity without `level`, msg None without
`message`, and one "_" + name (+ the type's suffix) pair per part, typed by the schema.  GPU only."""
import re

import numpy as np
import pytest

import vectors as V

pytestmark = pytest.mark.gpu
LTSV = 1
INVALID_UTF8 = 76
FLAG_MISSING_VALUE = 0x02
# bench.py's schema and suffixes, plus two names that compose to the same key: x:1 -> "_x_u64", x_u64:2 -> "_x_u64"
TYPED_SCHEMA = {"counter": "u64", "score": "i64", "mean": "f64", "done": "bool", "x": "u64", "x_u64": "u64", "big": "u64",
                "neg": "i64"}
SUFFIXES = {"u64": "_u64", "i64": "_i64", "f64": "_f64", "bool": "_bool"}
CONFIGS = {"untyped": (None, None), "typed": (TYPED_SCHEMA, SUFFIXES), "schema": (V.LTSV_SCHEMA, None),
           "g13": (V.LTSV_SCHEMA_G13, V.LTSV_SUFFIX_G13), "g14": (V.LTSV_SCHEMA_G14, V.LTSV_SUFFIX_G14)}
# extras replace fixed keys and the pair "_x", and add keys an LTSV Record leaves out: extras are always written
EXTRAS = [None, {"_x": "extra", "level": "9", "sd_id": "id\\1", "application_name": "app"}]
LTSV_ERRORS = ["Unable to parse the English to Unix timestamp in LTSV decoder", "Invalid severity level",
               "Severity level should be <= 7", "Type error; boolean was expected", "Type error; f64 was expected",
               "Type error; i64 was expected", "Type error; u64 was expected", "Missing timestamp", "Missing hostname"]

T = b"time:1\thost:h"
EDGES = [
    T, T + b"\tmessage:", T + b"\tmessage:m", b"time:1\thost:", b"time:1\thost:\tmessage:",          # None vs Some("")
    b"time:1\ttime:2\thost:a\thost:b\tlevel:1\tlevel:3\tmessage:a\tmessage:b",                     # repeated fixed keys
    T + b"\tx:1\ty:a\tx:2\tx:3\ty:b", T + b"\tx:1\tx_u64:2", T + b"\tx_u64:2\tx:1",                # duplicates, collisions
    T + b"\tcounter:1\tcounter_u64:s\tcounter_u64_u64:t", T + b"\tdone:true\tdone_bool:x\tdone:false",
    b"time:inf\thost:h", b"time:-inf\thost:h", b"time:nan\thost:h", b"time:-0.0\thost:h", b"time:1e21\thost:h",
    b"time:1e-7\thost:h", b"time:5e-324\thost:h", b"time:2.2250738585072011e-308\thost:h",
    T + b"\tmean:inf\tm2:x", T + b"\tmean:-inf", T + b"\tmean:NaN", T + b"\tmean:-0.0", T + b"\tmean:0",
    T + b"\tmean:1e21", T + b"\tmean:1e20", T + b"\tmean:1e-7", T + b"\tmean:1e-6", T + b"\tmean:5e-324",
    T + b"\tmean:2.2250738585072011e-308", T + b"\tmean:0.1", T + b"\tmean:123456789012345678901234567890",
    T + b"\tneg:-9223372036854775808", T + b"\tbig:18446744073709551615", T + b"\tcounter:+7\tscore:+0009\tneg:-0",
    T + b"\tcounter:007\tscore:-12\tbig:0", T + b"\tscore:9223372036854775807",
    b'time:1\thost:h"q\\\tk"e\\y:v"\\\x01w\tmessage:\xc3\xa9\xe6\x97\xa5\xf0\x9f\x9a\x80"\\\x01\x1f\ttab\x08:\x0c\r',
    "time:1\thost:日本\tnäme:ü\tместо:ʼ".encode(),
    b"foo\ttime:1\thost:h\tbar", b"time:1\thost:h\t\t\t", b"foo\tlevel:9\tbar", b"a\tb\ttime:x\tc\thost:h",
    b"foo\tdone:maybe\tbar\thost:h\ttime:1", b"\t", b"", b"nothing", b"a\tb:c\td",
    T + b"\tlevel:0", T + b"\tlevel:7\tlevel:8",
]


def _many(k: int, typed: bool = True) -> bytes:
    """a line of k pairs: repeated names, typed values, names that sort around the fixed keys and the extras"""
    parts = [b"time:1", b"host:h"]
    for j in range(k):
        nm = [b"a%02d" % (j % 17), b"x", b"counter", b"_x", b"zz%d" % j, b"level_", b"host2"][j % 7]
        val = b"%d" % (j * 7919) if (typed and nm in (b"x", b"counter")) else b'v"%d\\' % j
        parts.append(nm + b":" + val)
    return b"\t".join(parts + [b"message:end"])


LONG = [_many(25), _many(30), _many(60), _many(200), _many(1000)]


def _cfg(oracle, name):
    schema, suffixes = CONFIGS[name]
    if schema is None and suffixes is None:
        return None
    return oracle.LtsvConfig(schema, suffixes)


def _decoder(native, name, **kw):
    schema, suffixes = CONFIGS[name]
    return native.BatchDecoder(LTSV, ltsv_schema=schema, ltsv_suffixes=suffixes, **kw)


def _arr(b: bytes) -> np.ndarray:
    return np.frombuffer(b, dtype=np.uint8).copy() if b else np.zeros(0, np.uint8)


def _same_records(buf, offs, ebuf, eo, lines):
    if buf == ebuf and np.array_equal(offs, eo):
        return
    for i in range(len(eo) - 1):
        got, want = buf[offs[i]:offs[i + 1]], ebuf[eo[i]:eo[i + 1]]
        assert got == want, (i, lines[i][:200], got[:400], want[:400])
    raise AssertionError("record extents differ")


def _want_stops(res, offs):
    """what the non-fused path replays from fg_decode_batch (flowgger.cpp materialize_record): the failing part's offset
    on an error row, the line's length + 1 otherwise, -1 without FG_FLAG_MISSING_VALUE or for a line that is not UTF-8"""
    meta = res.meta.astype(np.int64)
    st, flags = meta & 0xFF, (meta >> 24) & 0xFF
    full = res.full_msg.astype(np.int64)
    lo = offs[:-1].astype(np.int64)
    stop = np.where(st != 0, full[:, 0] - lo, np.diff(offs).astype(np.int64) + 1)
    return np.where(((flags & FLAG_MISSING_VALUE) != 0) & (st != INVALID_UTF8), stop, -1).astype(np.int32)


def replay(line: bytes, stop: int) -> list[bytes]:
    """ltsv_decoder.rs:99 from a stop: the parts without ':' that start before it"""
    out, a = [], 0
    if stop < 0:
        return out
    for part in line.split(b"\t"):
        if a >= stop:
            break
        if b":" not in part:
            out.append(b"Missing value for name '" + part + b"'")
        a += len(part) + 1
    return out


_OUT = re.compile(rb";out=(\d+)")


def check(dec, oracle, lines, cfg_name, extra=None):
    """fg_decode_encode_gelf on pre-framed lines against the oracle; statuses against fg_decode_batch; stops against
    fg_decode_batch's rows and their replay against the oracle's count of println! lines.  Returns (records, statuses,
    stops)."""
    cfg = _cfg(oracle, cfg_name)
    dec.set_gelf_extra(extra or {})
    d, o = oracle.pack(lines)
    buf, offs, st, _ = dec.decode_encode_gelf(d, o)
    stops = dec.ltsv_stops()
    ebuf, eo = oracle.decode_encode_gelf(LTSV, d, o, extra or {}, cfg=cfg, nthreads=16)
    _same_records(buf, offs, ebuf, eo, lines)
    res = dec.decode(d, o)
    assert np.array_equal(st, (res.meta & 0xFF).astype(np.uint8))
    assert np.array_equal(stops, _want_stops(res, o))
    dump, do = oracle.decode_dump(LTSV, d, o, cfg, nthreads=16)
    for i, l in enumerate(lines):
        m = _OUT.search(dump[do[i]:do[i + 1]])
        assert len(replay(l, int(stops[i]))) == int(m.group(1)), (i, l[:200], stops[i])
    return [buf[offs[i]:offs[i + 1]] for i in range(len(lines))], st, stops


@pytest.fixture(scope="module", params=sorted(CONFIGS))
def cfg_dec(request, native):
    d = _decoder(native, request.param, max_batch_bytes=96 << 20, max_batch_lines=1 << 20)
    yield request.param, d
    d.close()


GOLDEN = [V.G9_LINE, V.G10_LINE, V.G11_LINE, V.G12_LINE, V.G13_LINE, V.G14_LINE]


@pytest.mark.parametrize("extra", EXTRAS, ids=["plain", "gelf_extra"])
def test_goldens_and_cases(cfg_dec, native, oracle, extra):
    name, dec = cfg_dec
    lines = [l.encode() for l in GOLDEN] + [l.encode() for l, _ in V.LTSV_CASES] + [l.encode() for l, _ in V.LTSV_SCHEMA_CASES]
    recs, st, stops = check(dec, oracle, lines, name, extra)
    errs = {native.error_string(LTSV, int(s)) for s in st if s}
    want_errs = set(LTSV_ERRORS) if name in ("schema", "typed", "g13") else set(LTSV_ERRORS[:3] + LTSV_ERRORS[-2:])
    assert want_errs <= errs, want_errs - errs
    assert (stops >= 0).sum() > 0
    ok = st == 0
    good = [r for r, g in zip(recs, ok) if g]
    assert all(r == b"" for r, g in zip(recs, ok) if not g)
    if extra is None:
        assert not any(k in r for r in good for k in (b'"application_name"', b'"process_id"', b'"sd_id"'))
        assert all(b'"full_message":' in r for r in good)
    else:
        assert all(b'"level":"9"' in r and b'"application_name":"app"' in r and b'"sd_id":"id\\\\1"' in r for r in good)
    if name in ("g13", "g14"):  # G13 with its suffixes, and G14 whose names already end in them, give the same pairs
        rec = recs[4] if name == "g13" else recs[5]
        assert all(k in rec for k in (b'"_done_bool":true', b'"_score_i64":-1', b'"_mean_f64":0.42', b'"_counter_u64":42'))


@pytest.mark.parametrize("extra", EXTRAS, ids=["plain", "gelf_extra"])
def test_edges(cfg_dec, oracle, extra):
    name, dec = cfg_dec
    recs, st, stops = check(dec, oracle, EDGES + LONG, name, extra)
    assert all(len(recs[len(EDGES) + k]) > 0 for k in range(len(LONG)))
    if extra is None:
        assert b'"short_message":"-"' in recs[0] and b'"short_message":""' in recs[1]
        assert b'"host":"unknown"' in recs[3]
    if name == "typed" and extra is None:
        r = dict(zip(EDGES, recs))
        assert b'"_x_u64":2' in r[T + b"\tx:1\tx_u64:2"] and r[T + b"\tx:1\tx_u64:2"].count(b'"_x_u64"') == 1
        assert b'"_x_u64":1' in r[T + b"\tx_u64:2\tx:1"]
        assert b'"_counter_u64":7,' in r[T + b"\tcounter:+7\tscore:+0009\tneg:-0"]
        assert b'"_neg_i64":-9223372036854775808' in r[T + b"\tneg:-9223372036854775808"]
        assert b'"_big_u64":18446744073709551615' in r[T + b"\tbig:18446744073709551615"]
        assert b'"_mean_f64":null' in r[T + b"\tmean:inf\tm2:x"] and b'"timestamp":null' in r[b"time:inf\thost:h"]
    assert [replay(l, int(s)) for l, s in zip(EDGES, stops)][EDGES.index(b"time:1\thost:h\t\t\t")] == [b"Missing value for name ''"] * 3


def test_generated_prefamed_and_split(native, oracle):
    """200 k bench-shaped lines, typed and untyped: against the oracle, and the split call against the pre-framed one"""
    data, offs = native.generate(LTSV, 1757, 200_000, bad_frac=0.02)
    lines = [bytes(data[offs[i]:offs[i + 1]]) for i in range(200_000)]
    rng = np.random.default_rng(1757)
    for name in ("untyped", "typed"):
        dec = _decoder(native, name, max_batch_bytes=128 << 20, max_batch_lines=1 << 20)
        try:
            for extra in EXTRAS:
                recs, st, stops = check(dec, oracle, lines, name, extra)
                assert (st == 0).sum() > 190_000
                parts = [l + (b"\r\n" if rng.random() < 0.1 else b"\n") for l in lines]
                sbuf, so, sst, sl, _ = dec.split_decode_encode_gelf(_arr(b"".join(parts)), 0)
                assert b"".join(recs) == sbuf and np.array_equal(np.diff(so), [len(r) for r in recs])
                assert np.array_equal(sst, st) and np.array_equal(dec.ltsv_stops(), stops)
        finally:
            dec.close()


def _frame(stream: bytes, framing: int):
    import pysplit
    return (pysplit.split_nul if framing else pysplit.split_lines)(stream)


def check_split(dec, oracle, stream: bytes, framing: int, cfg_name: str, extra=None):
    """fg_split_decode_encode_gelf against the host framing + the oracle; invalid records: status 76, no bytes, no stop;
    the pre-framed call on the valid records gives the same records, statuses and stops"""
    dec.set_gelf_extra(extra or {})
    buf, o, status, line_offs, _ = dec.split_decode_encode_gelf(_arr(stream), framing)
    stops = dec.ltsv_stops()
    offs, lines, valid = _frame(stream, framing)
    n = len(lines)
    assert np.array_equal(line_offs, offs) and len(status) == n and len(stops) == n
    valid = np.asarray(valid, dtype=bool)
    good = [l for l, v in zip(lines, valid) if v]
    d, do = oracle.pack(good)
    ebuf, eo = oracle.decode_encode_gelf(LTSV, d, do, extra or {}, cfg=_cfg(oracle, cfg_name), nthreads=16)
    want_len = np.zeros(n, np.int64)
    want_len[valid] = np.diff(eo)
    assert buf == ebuf and np.array_equal(np.diff(o), want_len)
    assert np.all(status[~valid] == INVALID_UTF8) and np.all(stops[~valid] == -1)
    pbuf, po, pst, _ = dec.decode_encode_gelf(d, do)
    assert pbuf == buf and np.array_equal(po, eo) and np.array_equal(pst, status[valid])
    assert np.array_equal(dec.ltsv_stops(), stops[valid])
    return n


G = b"time:1\thost:h\tfoo\tk:v"
LINE_EDGES = [b"", b"\n", b"\n\n", G, G + b"\n", G + b"\r\n", G + b"\r", b"\r\n" + G, G + b"\n\n" + G + b"\n",
              b"\xff\n" + G + b"\n", G + b"\n\xc3", G + b"\n\xc3\n\xa9" + G + b"\n", b"foo\tbar\xff\n" + G,
              b"\n".join(EDGES) + b"\n", b"\r\n".join(LONG)]
NUL_EDGES = [b"", b"\0", b"\0\0", G, G + b"\0", G + b"\r\n\0", G + b"\0\0" + G + b"\0", b"\xff\0" + G + b"\0", G + b"\0\xc3",
             G + b"\n" + G + b"\0", b"\0".join(EDGES)]


@pytest.mark.parametrize("extra", EXTRAS, ids=["plain", "gelf_extra"])
def test_split_framing_edges(cfg_dec, oracle, extra):
    name, dec = cfg_dec
    for stream in LINE_EDGES:
        check_split(dec, oracle, stream, 0, name, extra)
    for stream in NUL_EDGES:
        check_split(dec, oracle, stream, 1, name, extra)


def test_split_three_chunks(native, oracle):
    """More than 128 MiB: records straddle both 64 MiB chunk boundaries with a multi-byte character, a truncated
    sequence or a CRLF cut in two"""
    prefix = b"time:1\thost:h\tnm\tname:"
    line = prefix + b"7" * (63 - len(prefix)) + b"\n"
    B = 64 << 20

    def to(cur, start, parts):
        gap = start - cur
        k = gap // 64 - 1
        parts.append(line * k)
        parts.append(prefix + b"8" * (gap - 64 * k - len(prefix) - 1) + b"\n")
        return start

    d = _decoder(native, "typed", max_batch_bytes=160 << 20, max_batch_lines=3 << 20)
    try:
        for specials in [(("日".encode(), 1), (b"\xe2\x82", 1)), (("\U0001F680".encode(), 3), (b"\r", 1))]:
            parts, cur = [], 0
            for b, (tail, before) in zip((B, 2 * B), specials):
                special = prefix + b"1\ts:" + tail + b"\n"
                cur = to(cur, b - len(prefix) - 4 - before, parts)
                parts.append(special)
                cur += len(special)
            parts.append(line * 1000 + prefix + b"9")
            stream = b"".join(parts)
            assert len(stream) > 2 * B
            check_split(d, oracle, stream, 0, "typed")
    finally:
        d.close()


# 1 MiB / 1024-line context: the side table starts at 43690 rows, the output buffer at 2 x 1 MiB + 200 B per line
PAIR_LINES = [b"time:1\thost:h\t" + b"\t".join(b"k%d:v" % j for j in range(60)) + b"\tx:1\tlonely"] * 1000  # 62 k rows
OUTPUT_LINES = [b"time:1\thost:h\tmessage:" + b'\\"' * 490] * 900                        # every byte escaped, twice per record


@pytest.mark.parametrize("lines", [PAIR_LINES, OUTPUT_LINES], ids=["side-table", "output-buffer"])
@pytest.mark.parametrize("split", [True, False], ids=["split", "framed"])
def test_regrow(native, oracle, lines, split):
    cfg = _cfg(oracle, "typed")
    ebuf, eo = oracle.decode_encode_gelf(LTSV, *oracle.pack(lines), {}, cfg=cfg, nthreads=16)
    assert len(eo) == len(lines) + 1 and np.all(np.diff(eo) > 0)
    if lines is OUTPUT_LINES:
        assert len(ebuf) > 2 * (1 << 20) + 1024 * 200
    stream = _arr(b"\n".join(lines) + b"\n")
    dd, do = oracle.pack(lines)
    d = _decoder(native, "typed", max_batch_bytes=1 << 20, max_batch_lines=1024)
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
            want = np.full(len(lines), len(lines[0]) + 1 if lines is PAIR_LINES else -1, np.int32)
            assert np.array_equal(d.ltsv_stops(), want)
        assert launches[0] == 2 * launches[1], launches  # the first call overflowed and redid the batch once
        # the context's next call, on other lines, against the oracle and a fresh context
        small = EDGES + LONG
        recs, st, stops = check(d, oracle, small, "typed")
        f = _decoder(native, "typed", max_batch_bytes=1 << 20, max_batch_lines=1024)
        try:
            fr, fs, fstops = check(f, oracle, small, "typed")
        finally:
            f.close()
        assert recs == fr and np.array_equal(st, fs) and np.array_equal(stops, fstops)
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


def test_refused_inputs_leave_the_context_usable(native, oracle):
    """GELF input on an LTSV context, and LTSV input on a context created for another input.format, are refused by both
    fused calls with the same text (and leave no stops); the contexts then work as before"""
    refused = "the fused encoder takes input.format = rfc5424"
    d = _decoder(native, "typed", max_batch_bytes=1 << 20, max_batch_lines=1 << 12)
    r5 = native.BatchDecoder(native.FMT_RFC5424, max_batch_bytes=1 << 20, max_batch_lines=1 << 12)
    try:
        check(d, oracle, EDGES, "typed")
        for split in (True, False):
            assert _raw_fused(d, native.FMT_GELF, b'{"host":"h","short_message":"m"}\n', split) == (-1, refused)
            with pytest.raises(RuntimeError, match="fg_encoded_ltsv_stops"):
                d.ltsv_stops()
            assert _raw_fused(r5, native.FMT_LTSV, G + b"\n", split) == (-1, refused)
        check(d, oracle, EDGES, "typed")
        check_split(d, oracle, b"\n".join(EDGES), 0, "typed")
        dd, do = oracle.pack([V.G1_LINE.encode(), V.G2_LINE.encode()])
        buf, offs, st, _ = r5.decode_encode_gelf(dd, do)
        ebuf, eo = oracle.decode_encode_gelf(0, dd, do, {}, nthreads=2)
        assert buf == ebuf and np.array_equal(offs, eo) and np.all(st == 0)
    finally:
        d.close()
        r5.close()


def _splitter_records(native, framing):
    data, offs = native.generate(LTSV, 17, 3000, bad_frac=0.02)
    lines = [bytes(data[offs[i]:offs[i + 1]]) for i in range(3000)]
    lines[5] = lines[5] + b"\r"
    lines[6] = b"time:1\thost:h\tfoo\t\xff\xfe broken utf8"
    lines[7] = lines[7] + b"\xe2\x82"
    lines[8] = b""
    lines[9] = b"   "
    lines[12:12 + len(EDGES)] = EDGES
    lines[1000] = b"time:1\thost:h\tmiss\tmessage:" + b"y " * (3 << 19)          # longer than the 1 MiB context
    if framing == 2:  # syslen: a record that is not UTF-8 ends the stream
        lines[6] = b"time:1\thost:h\tfoo\tfine"
        lines[7] = lines[7][:-2]
    return lines[:2000] + [b"x"] * 50_000 + lines[2000:]


def _splitter_text(recs, framing):
    if framing == 2:
        return b"".join(b"%d %s" % (len(r), r) for r in recs)
    d = b"\0" if framing else b"\n"
    return d.join(recs) + d


@pytest.mark.parametrize("cfg_name", ["untyped", "typed"])
@pytest.mark.parametrize("framing", [0, 1, 2], ids=["line", "nul", "syslen"])
def test_splitters_end_to_end(native, oracle, framing, cfg_name):
    """records against the oracle's encoder; stderr and stdout identical to the non-fused splitter on the same input"""
    recs = _splitter_records(native, framing)
    text = _splitter_text(recs, framing)
    if framing == 2:
        lines, valid = recs, [True] * len(recs)
    else:
        _, lines, valid = _frame(text, framing)
    good = [l for l, v in zip(lines, valid) if v]
    d, o = oracle.pack(good)
    ebuf, eo = oracle.decode_encode_gelf(LTSV, d, o, {"env": "prod"}, cfg=_cfg(oracle, cfg_name), nthreads=16)
    want = [ebuf[eo[k]:eo[k + 1]] for k in range(len(good)) if eo[k + 1] > eo[k]]
    dec = _decoder(native, cfg_name, max_batch_bytes=1 << 20, max_batch_lines=1 << 12)
    try:
        records, err, out = native.splitter_run_gelf(dec, text, {"env": "prod"}, max_lines=1 << 16, max_bytes=1 << 20,
                                                     framing=framing, stdout=True)
        assert records.split(b"\n")[:-1] == want
        _, err2, out2 = native.splitter_run(dec, text, max_lines=1 << 16, max_bytes=1 << 20, framing=framing)
        assert err == err2
        assert out == out2 and out.count(b"Missing value for name") > 50_000
    finally:
        dec.close()
