"""output.framing on the device: the fused GELF calls (fg_decode_encode_gelf, fg_split_decode_encode_gelf) with
fg_set_output_framing return the bytes the reference's Output writes, the merger (merger/*.rs) applied to every record
GelfEncoder::encode returns, and nothing for a record the decoder or the UTF-8 check rejected.  The expected stream is
the merger restatement (tests/merger_oracle.py) over the decode + encode oracle's records; statuses are the unframed
call's.  GPU only."""
import hashlib
import os

import numpy as np
import pytest

import merger_oracle as M
import vectors as V

pytestmark = pytest.mark.gpu
R5, LTSV, GELF, R3 = 0, 1, 2, 3
YEAR = 2026  # RFC3164: the year of a timestamp without one, fixed on both sides
INVALID_UTF8 = 76
FLAG_TS_MISSING = 0x01
FG_E_ARG = -1
NTHREADS = os.cpu_count() or 8
FRAMINGS = {"line": M.LINE, "nul": M.NUL, "syslen": M.SYSLEN}
TYPED = {"counter": "u64", "score": "i64", "mean": "f64", "done": "bool"}
SUFFIXES = {"u64": "_u64", "i64": "_i64", "f64": "_f64", "bool": "_bool"}
SOURCES = {"rfc5424": R5, "rfc3164": R3, "ltsv": LTSV, "ltsv_typed": LTSV, "gelf": GELF}
SEEDS = {"rfc5424": 5, "rfc3164": 3, "ltsv": 1, "ltsv_typed": 11, "gelf": 2}
BAD = b"\xff\xfe not UTF-8"


def framed_len(n: int, framing: int) -> int:
    if framing == M.SYSLEN:
        return len(str(n + 1)) + 1 + n + 1
    return n + (0 if framing == M.NONE else 1)


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


def _arr(b: bytes) -> np.ndarray:
    return np.frombuffer(b, dtype=np.uint8).copy() if b else np.zeros(0, np.uint8)


class Expected:
    """The oracle's GELF records of a source's lines (b"" for a rejected line).  A GELF record without "timestamp" gets
    the call's clock (fg_encoded_gelf_now): the oracle leaves its Record.ts at 0.0, replaced per call."""

    def __init__(self, oracle, dec, src, lines):
        self.lines = lines
        d, o = oracle.pack(lines)
        buf, eo = oracle.decode_encode_gelf(SOURCES[src], d, o, cfg=_cfg(oracle, src), nthreads=NTHREADS)
        self.recs = [buf[eo[i]:eo[i + 1]] for i in range(len(lines))]
        self.missing = []
        if src == "gelf":
            meta = dec.decode(d, o).meta.astype(np.int64)
            self.missing = np.flatnonzero(((meta & 0xFF) == 0) & (((meta >> 24) & FLAG_TS_MISSING) != 0)).tolist()
        self.oracle = oracle

    def records(self, now=None):
        if not self.missing:
            return self.recs
        at = b',"timestamp":' + self.oracle.format_f64(now).encode() + b','
        recs = list(self.recs)
        for i in self.missing:
            recs[i] = recs[i].replace(b',"timestamp":0.0,', at)
        return recs


def _source_lines(native, src, n):
    """vectors + n generated lines with decoder rejects; no line holds a terminator of either input framing"""
    data, offs = native.generate(SOURCES[src], SEEDS[src], n, bad_frac=0.02)
    lines = [l.encode() for l in _vector_lines(src)] + [bytes(data[offs[i]:offs[i + 1]]) for i in range(n)]
    return [l for l in lines if b"\n" not in l and b"\r" not in l and b"\0" not in l]


@pytest.fixture(scope="module", params=sorted(SOURCES))
def source(request, native, oracle):
    src = request.param
    dec = _decoder(native, src, max_batch_bytes=64 << 20, max_batch_lines=1 << 18)
    lines = _source_lines(native, src, 100_000)
    exp = Expected(oracle, dec, src, lines)
    yield src, dec, exp
    dec.close()


def _run(dec, call, lines, bad=True):
    """one fused call: (bytes, offsets, status, ok-line index per record or None for an invalid one, clock)"""
    if call == "prefamed":
        d, o = _pack(lines)
        buf, offs, st, _ = dec.decode_encode_gelf(d, o)
        which = list(range(len(lines)))
    else:
        # with `bad`, a record that is not UTF-8 before every 997th line: "Invalid UTF-8 input", no record
        delim = b"\n" if call == "line" else b"\0"
        parts, which = [], []
        for i, l in enumerate(lines):
            if bad and i % 997 == 500:
                parts.append(BAD)
                which.append(None)
            parts.append(l)
            which.append(i)
        buf, offs, st, _, _ = dec.split_decode_encode_gelf(_arr(delim.join(parts) + delim), 0 if call == "line" else 1)
        assert len(st) == len(which)
    now = dec.gelf_now() if dec.fmt == GELF else None
    return buf, offs, st, which, now


def _pack(lines):
    offs = np.zeros(len(lines) + 1, np.int32)
    np.cumsum([len(l) for l in lines], out=offs[1:])
    return _arr(b"".join(lines)), offs


def _check(dec, exp, call, framing):
    dec.set_output_framing(M.NONE)
    _, _, ust, _, _ = _run(dec, call, exp.lines)
    dec.set_output_framing(framing)
    buf, offs, st, which, now = _run(dec, call, exp.lines)
    dec.set_output_framing(M.NONE)
    assert np.array_equal(st, ust)
    recs = exp.records(now)
    got = [recs[i] if i is not None else b"" for i in which]
    ok = [bool(r) for r in got]
    assert [bool(s == 0) for s in st] == ok
    assert all(st[k] == INVALID_UTF8 for k, i in enumerate(which) if i is None)
    want = M.output_stream(got, ok, framing)
    lens = np.diff(offs)
    want_lens = np.array([framed_len(len(r), framing) if g else 0 for r, g in zip(got, ok)], np.int64)
    if buf != want or not np.array_equal(lens, want_lens):
        for k, (r, g) in enumerate(zip(got, ok)):
            w = M.MERGERS[framing](r) if g else b""
            assert buf[offs[k]:offs[k + 1]] == w, (k, which[k], buf[offs[k]:offs[k + 1]][:300], w[:300])
        raise AssertionError("record extents differ")


@pytest.mark.parametrize("call", ["prefamed", "line", "nul"])
@pytest.mark.parametrize("framing", sorted(FRAMINGS))
def test_every_framing_source_and_call(source, call, framing):
    src, dec, exp = source
    _check(dec, exp, call, FRAMINGS[framing])


def test_none_is_todays_output(native, oracle):
    """FG_OUT_NONE, set explicitly or after another framing, gives the bytes and offsets of a context that never set it"""
    lines = _source_lines(native, "rfc5424", 20_000)
    d, o = _pack(lines)
    stream = _arr(b"\n".join(lines) + b"\n")
    results = []
    for setup in ([], [M.NONE], [M.SYSLEN, M.NONE], [M.LINE, M.NUL, M.NONE]):
        dec = _decoder(native, "rfc5424", max_batch_bytes=16 << 20, max_batch_lines=1 << 16)
        try:
            for f in setup:
                dec.set_output_framing(f)
                if f != M.NONE:
                    dec.decode_encode_gelf(d, o)
            results.append((dec.decode_encode_gelf(d, o)[:3], dec.split_decode_encode_gelf(stream)[:3]))
        finally:
            dec.close()
    for r in results[1:]:
        for (b0, o0, s0), (b1, o1, s1) in zip(results[0], r):
            assert b0 == b1 and np.array_equal(o0, o1) and np.array_equal(s0, s1)


def test_syslen_digit_edges(native, oracle):
    """Records whose length + 1 is 99, 100, 999, 1000, 9999, 10000 and 100000, each started at output offsets of every
    residue mod 4.  (A GELF record is longer than 10 bytes: the prefixes of 9 and 10 are checked by test_emu_out_framing.)"""
    def line(k):
        return b'{"host":"h","short_message":"' + b"m" * k + b'","timestamp":1}'
    d, o = _pack([line(0)])
    c = len(oracle.decode_encode_gelf(GELF, d, o)[0])  # record length of line(k) = c + k
    lines, edges, at = [], [], 0  # `at`: output offset of the next record
    for target in (99, 100, 999, 1000, 9999, 10000, 100000):
        for residue in range(4):  # a filler record of c + pad bytes in front moves this copy's start to `residue` mod 4
            pad = next(p for p in range(4) if (at + framed_len(c + p, M.SYSLEN)) % 4 == residue)
            lines.append(line(pad))
            at += framed_len(c + pad, M.SYSLEN)
            edges.append(len(lines))
            lines.append(line(target - 1 - c))
            at += framed_len(target - 1, M.SYSLEN)
    dec = _decoder(native, "gelf", max_batch_bytes=8 << 20, max_batch_lines=1 << 12)
    try:
        exp = Expected(oracle, dec, "gelf", lines)
        assert [len(exp.recs[i]) + 1 for i in edges[::4]] == [99, 100, 999, 1000, 9999, 10000, 100000]
        for call in ("prefamed", "line", "nul"):
            dec.set_output_framing(M.SYSLEN)
            buf, offs, st, which, now = _run(dec, call, lines)
            assert buf == M.output_stream(exp.records(now), [True] * len(lines), M.SYSLEN)
            for g in range(0, len(edges), 4):  # the four copies of each edge length start at every residue mod 4
                assert {int(offs[which.index(i)]) % 4 for i in edges[g:g + 4]} == {0, 1, 2, 3}
            for i in edges:
                k = which.index(i)
                assert buf[offs[k]:offs[k + 1]].startswith(b"%d " % (len(exp.recs[i]) + 1))
    finally:
        dec.close()


def test_stream_past_one_chunk(native, oracle):
    """A raw stream of more than one 64 MiB chunk of split_stream: frames stay whole across the steps"""
    n = 190_000
    data, offs = native.generate(R5, 64, n, mean_len=400.0, bad_frac=0.01, nthreads=NTHREADS, terminated=True)
    stream = np.asarray(data)
    assert len(stream) > (64 << 20)
    lines = [bytes(stream[offs[i]:offs[i + 1] - 1]) for i in range(n)]
    d, o = _pack(lines)
    ebuf, eo = oracle.decode_encode_gelf(R5, d, o, nthreads=NTHREADS)
    recs = [ebuf[eo[i]:eo[i + 1]] for i in range(n)]
    dec = _decoder(native, "rfc5424", max_batch_bytes=len(stream) + (1 << 20), max_batch_lines=n + 64)
    try:
        for framing in (M.NUL, M.SYSLEN):
            dec.set_output_framing(framing)
            buf, boffs, st, lo, _ = dec.split_decode_encode_gelf(stream)
            assert np.array_equal(lo, offs)
            assert buf == M.output_stream(recs, [bool(r) for r in recs], framing)
            assert np.array_equal(np.diff(boffs), [framed_len(len(r), framing) if r else 0 for r in recs])
    finally:
        dec.close()


@pytest.mark.parametrize("call", ["prefamed", "line"])
def test_regrow_by_frame_bytes_alone(native, oracle, call):
    """The context's first output buffer (2 x max_batch_bytes + 200 B per line, in 4 KiB pages) holds the unframed
    records but not the framed ones: the framed call regrows it and redoes the batch; the unframed one does not."""
    n = 5056
    N = n + 64  # max_batch_lines, a multiple of 64 as the context keeps it (a split call takes fewer than N lines)
    lines = [b"<13>1 2015-08-05T15:53:45Z h%05d a p m - %s" % (i, b'"' * 100) for i in range(n)]  # every '"' escaped twice
    d, o = _pack(lines)
    ebuf, eo = oracle.decode_encode_gelf(R5, d, o, nthreads=NTHREADS)
    U = len(ebuf)
    cap = -(-U // 4096) * 4096
    assert U <= cap < U + n  # one frame byte per record (line framing) is more than the slack
    B = (cap - 200 * N) // 2
    assert B >= int(o[-1]) + n and (2 * B + 200 * N + 4095) // 4096 * 4096 == cap
    launches = {}
    for framing in (M.NONE, M.LINE):
        dec = _decoder(native, "rfc5424", max_batch_bytes=B, max_batch_lines=N)
        try:
            dec.set_output_framing(framing)
            buf, offs, st, which, _ = _run(dec, call, lines, bad=False)
            recs = [ebuf[eo[i]:eo[i + 1]] for i in range(n)]
            assert all(recs) and all(i is not None for i in which)
            assert buf == M.output_stream(recs, [True] * n, framing)
            launches[framing] = dec.kernel_launches()
        finally:
            dec.close()
    assert launches[M.LINE] > launches[M.NONE]


def test_one_launch_past_4gib(native, oracle):
    """One syslen-framed launch whose output passes 2^32 bytes (512 Ki escape-heavy RFC5424 lines): offsets rise, the
    stream is the oracle's, and the prefix of the first record that starts past 2^32 is its length + 1"""
    n = 512 << 10
    msg = (b'"\\' * 9 + b"ab") * 115
    lines = (b"<13>1 %s host%07d a p m - %s" % (V.TS.encode(), i, msg) for i in range(n))
    line0 = b"<13>1 %s host%07d a p m - %s" % (V.TS.encode(), 0, msg)
    total = n * len(line0)
    data = np.empty(total, np.uint8)
    mv = memoryview(data)
    offs = np.arange(n + 1, dtype=np.int64) * len(line0)
    for i, l in enumerate(lines):
        mv[offs[i]:offs[i + 1]] = l
    offs = offs.astype(np.int32)
    dec = _decoder(native, "rfc5424", max_batch_bytes=total + (1 << 20), max_batch_lines=n + 64)
    try:
        dec.set_output_framing(M.SYSLEN)
        buf, boffs, st, _ = dec.decode_encode_gelf(data, offs, copy=False)
        assert (st == 0).all()
        assert (np.diff(boffs) > 0).all() and int(boffs[-1]) > (1 << 32) and len(buf) == int(boffs[-1])
        first = int(np.searchsorted(boffs, 1 << 32))
        step = 16 << 10
        for a in range(0, n, step):
            b = min(n, a + step)
            ebuf, eo = oracle.decode_encode_gelf(R5, data, offs[a:b + 1], nthreads=NTHREADS)
            recs = [ebuf[eo[i]:eo[i + 1]] for i in range(b - a)]
            want = M.output_stream(recs, [True] * len(recs), M.SYSLEN)
            got = buf[int(boffs[a]):int(boffs[b])]
            assert hashlib.blake2b(got).digest() == hashlib.blake2b(want).digest(), f"lines [{a}, {b})"
            if a <= first < b:
                r = recs[first - a]
                assert bytes(buf[int(boffs[first]):int(boffs[first]) + 8]).startswith(b"%d " % (len(r) + 1))
    finally:
        dec.close()


def _splitter_lines(native, src):
    data, offs = native.generate(SOURCES[src], 17, 20_000, bad_frac=0.02)
    return [bytes(data[offs[i]:offs[i + 1]]) for i in range(20_000)]


@pytest.mark.parametrize("src", ["rfc5424", "ltsv"])
@pytest.mark.parametrize("in_framing", [0, 1, 2], ids=["line", "nul", "syslen"])
def test_host_splitters(native, oracle, src, in_framing):
    """BatchingLineSplitter / BatchingNulSplitter / BatchingSyslenSplitter with device framing: the stream they send is
    the oracle's output stream, and their stderr / stdout are those of the unframed run"""
    lines = _splitter_lines(native, src)
    if in_framing == 2:  # syslen: a record that is not UTF-8 ends the stream
        text = b"".join(b"%d %s" % (len(l), l) for l in lines)
    else:  # one record that is not UTF-8: "Invalid UTF-8 input" on stderr, nothing sent
        delim = b"\0" if in_framing else b"\n"
        text = delim.join(lines[:100] + [BAD] + lines[100:]) + delim
    d, o = _pack(lines)
    ebuf, eo = oracle.decode_encode_gelf(SOURCES[src], d, o, nthreads=NTHREADS)
    recs = [ebuf[eo[i]:eo[i + 1]] for i in range(len(lines))]
    ok = [bool(r) for r in recs]
    assert not all(ok)
    dec = _decoder(native, src, max_batch_bytes=1 << 20, max_batch_lines=1 << 12)
    try:
        plain, err0, out0 = native.splitter_run_gelf(dec, text, max_lines=1 << 16, max_bytes=1 << 20, framing=in_framing, stdout=True)
        assert plain.split(b"\n")[:-1] == [r for r in recs if r]
        for framing in FRAMINGS.values():
            stream, err, out = native.splitter_run_gelf_framed(dec, text, framing, max_lines=1 << 16, max_bytes=1 << 20,
                                                               framing=in_framing)
            assert stream == M.output_stream(recs, ok, framing)
            assert err == err0 and out == out0
        stream, err, out = native.splitter_run_gelf_framed(dec, text, M.NONE, max_lines=1 << 16, max_bytes=1 << 20,
                                                           framing=in_framing)
        assert stream == b"".join(recs) and err == err0 and out == out0
    finally:
        dec.close()


def test_unknown_framing_is_refused(native, oracle):
    lines = [V.G1_LINE.encode(), V.G2_LINE.encode()]
    d, o = _pack(lines)
    dec = _decoder(native, "rfc5424", max_batch_bytes=1 << 20, max_batch_lines=1 << 10)
    try:
        dec.set_output_framing(M.LINE)
        L = native.load_cuda()
        for bad in (4, -1, 99):
            assert L.fg_set_output_framing(dec.ctx, bad) == FG_E_ARG
        buf, offs, st, _ = dec.decode_encode_gelf(d, o)
        ebuf, eo = oracle.decode_encode_gelf(R5, d, o)
        assert buf == M.output_stream([ebuf[eo[0]:eo[1]], ebuf[eo[1]:eo[2]]], [True, True], M.LINE)
    finally:
        dec.close()
