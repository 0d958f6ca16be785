"""The fused LTSV encoder at its own edges, against the oracle's decoders and LTSVEncoder::encode restated
(tests/ltsv_oracle.py), statuses against fg_decode_batch:
  - GELF strings (every \\uXXXX, surrogate pairs, short escapes, raw UTF-8, newline-retry forms) as host, short_message,
    full_message, member names and member values: the unescape step of run_ltsv on the device;
  - records whose segment lists end on and around the window boundaries (56, 112, 168 segments), every kind of segment
    (ltsv_out_edges.KINDS) on the last segment of a window and on the first of the next, with and without
    output.ltsv_extra, and framed by the mergers;
  - lines of length class 63, a CTA span read from global memory, warps with a rejected line and a four-window record
    at every lane;
  - one launch whose output passes 2^32 bytes, records placed on 2^31 and 2^32 or across 2^32 by one byte;
  - spans longer than the segment length fields: a 2^29 + 13-byte value (LTSV output) and a 2^30 + 13-byte string (GELF
    output) come out whole; a GELF string with escapes that long fails the call.  GPU only."""
import hashlib
import os
import re
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest

import ltsv_oracle as LO
import ltsv_out_edges as E
import merger_oracle as M
from test_emu_ltsv_json import CPS, RETRY, _pairs, _short_bodies
from test_gpu_encode_sizes import E31, E32, LAUNCH_LINES, SLICE, _digest, _first, _pack, _tune

pytestmark = pytest.mark.gpu
R5, LTSV, GELF, R3 = 0, 1, 2, 3
YEAR = 2026
NTHREADS = os.cpu_count() or 8
EXTRA = {"_x": "a\tb:c", "y": "1"}


def _cfg(oracle, src):
    if src == LTSV:
        return oracle.LtsvConfig(E.TYPED, E.SUFFIXES)
    return oracle.Rfc3164Config(YEAR) if src == R3 else None


@pytest.fixture(scope="module")
def decs(native):
    made = {}

    def get(src, **kw):
        key = (src, tuple(sorted(kw.items())))
        if key not in made:
            made[key] = native.BatchDecoder(src, ltsv_schema=E.TYPED if src == LTSV else None,
                                            ltsv_suffixes=E.SUFFIXES if src == LTSV else None,
                                            rfc3164_year=YEAR if src == R3 else 0, **kw)
        return made[key]
    yield get
    for d in made.values():
        d.close()


def _check(dec, oracle, src, lines, extra=None, framing=M.NONE):
    """every record equals the oracle's (framed by the merger), every status fg_decode_batch's; returns the records"""
    d, o = oracle.pack(lines)
    dec.set_ltsv_extra(extra or {})
    dec.set_output_framing(framing)
    try:
        buf, offs, st, _ = dec.decode_encode_ltsv(d, o)
    finally:
        dec.set_output_framing(M.NONE)
        dec.set_ltsv_extra({})
    now = dec.gelf_now() if src == GELF else None
    want = LO.decode_encode_ltsv(oracle, src, d, o, extra=extra, cfg=_cfg(oracle, src), now=now, nthreads=NTHREADS)
    for i, w in enumerate(want):
        g = buf[offs[i]:offs[i + 1]]
        w = M.MERGERS[framing](w) if w else b""
        assert g == w, f"record {i}: line {lines[i][:300]!r}\n got  {g[:400]!r}\n want {w[:400]!r}"
    assert np.array_equal(st, dec.decode(d, o).status.astype(np.uint8))
    assert [bool(w) for w in want] == [s == 0 for s in st]
    return want


# ---- GELF strings on the device ----------------------------------------------------------------------------------------

def _bodies():
    esc = [b"\\u%04x" % c for c in CPS] + [b"ab:"[:c % 4] + b"\\u%04X" % c + b"xyz" for c in CPS]
    return esc + _pairs() + [b for b in _short_bodies() if b]


@pytest.mark.parametrize("where", ["host", "short_message", "full_message", "key", "value"])
def test_gelf_strings(decs, oracle, where):
    dec = decs(GELF, max_batch_bytes=64 << 20, max_batch_lines=1 << 18)
    if where in ("host", "short_message", "full_message"):
        lines = [b'{"host":"h","short_message":"m","timestamp":1,"' + where.encode() + b'":"' + b + b'"}' for b in _bodies()]
        lines = [l.replace(b'"host":"h",', b"", 1) if where == "host" else l for l in lines]
        lines = [l.replace(b'"short_message":"m",', b"", 1) if where == "short_message" else l for l in lines]
    elif where == "key":
        lines = [b'{"host":"h","short_message":"m","timestamp":1,"' + b + b'":"v"}' for b in _bodies()]
        lines += [b'{"host":"h","short_message":"m","timestamp":1,"' + p + b + b'":"v"}' for p in (b"_", b"\\u005f")
                  for b in _short_bodies()]
    else:
        lines = [b'{"host":"h","short_message":"m","timestamp":1,"_k":"' + b + b'"}' for b in _bodies()]
    want = _check(dec, oracle, GELF, lines)
    assert sum(bool(w) for w in want) >= 0.99 * len(lines)


def test_gelf_retry_lines(decs, oracle):
    """lines with a raw LF (the decoder's newline retry): strings in every place, raw LF and `\\` + LF"""
    dec = decs(GELF)
    lines = []
    for b in RETRY:
        lines += [b'{"host":"h\n","short_message":"' + b + b'","timestamp":1}',
                  b'{"host":"' + b + b'","short_message":"m","full_message":"' + b + b'","timestamp":1}',
                  b'{"host":"h","short_message":"m","timestamp":1,"_' + b + b'":"' + b + b'"}']
    want = _check(dec, oracle, GELF, lines)
    assert sum(map(bool, want)) >= 2 * len(lines) // 3  # (the decoder rejects some `\\` + LF forms outside short_message)


# ---- segment windows, tiles, lanes ------------------------------------------------------------------------------------

@pytest.mark.parametrize("framing", [M.NONE, M.SYSLEN, M.NUL])
@pytest.mark.parametrize("src", [R5, LTSV, GELF, R3])
def test_segment_windows(decs, oracle, src, framing):
    dec = decs(src)
    lines = E.window_lines(src)
    cells, totals = set(), set()
    d, o = oracle.pack(lines)
    buf, offs = oracle.decode_dump(src, d, o, cfg=_cfg(oracle, src), nthreads=NTHREADS)
    for extra in (None, EXTRA):
        want = _check(dec, oracle, src, lines, extra, framing)
        assert all(want)
        for i in range(len(lines)):
            seg = E.segments(LO.parse_dump(buf[offs[i]:offs[i + 1]], now=0.0), src, bool(extra))
            totals.add(len(seg))
            cells |= {(b, seg[b]) for b in E.BOUNDARIES if len(seg) > b}
    if src != R3:  # an RFC3164 record has no pairs: it never reaches a second window
        assert set(E.TOTALS) <= totals
        # every kind of segment the source emits sits on the last segment of the first and second window and on the
        # first segment of the second and third
        missing = {(b, k) for b in E.BOUNDARIES for k in E.KINDS[src]} - cells
        assert not missing, sorted(missing)


@pytest.mark.parametrize("framing", [M.NONE, M.SYSLEN, M.NUL])
@pytest.mark.parametrize("src", [R5, LTSV, GELF, R3])
def test_tiles_and_lanes(decs, oracle, src, framing):
    dec = decs(src)
    rng = np.random.default_rng(40 + src)
    _check(dec, oracle, src, E.long_lines(src, rng), EXTRA, framing)
    span = E.span_lines(src, rng)
    _, o = oracle.pack(span)
    assert int(o[256 * 5] - o[256 * 4]) > 4 * 32768  # above every encoder tile
    _check(dec, oracle, src, span, None, framing)
    want = _check(dec, oracle, src, E.lane_lines(src, rng), None, framing)
    assert sum(not w for w in want) == 32


# ---- one launch past 2^32 bytes of output -----------------------------------------------------------------------------

# An ~8.3 KB output.ltsv_extra makes every record of a ~41-byte RFC5424 line 8.4 KB: the 512 Ki lines of one launch
# (the default chunk_lines) pass 4 GiB of output from 21 MB of input.  One more fraction digit of the timestamp (the
# same Record.ts) is one more byte of full_message only, which places records exactly (_tune).
BIG_EXTRA = {"e": "x" * 8300}


def _big_line(extra: int) -> bytes:
    return b"<13>1 2015-08-05T15:53:45.5" + b"0" * extra + b"Z h a p id - m"


@pytest.mark.parametrize("framing,edges", [(M.NONE, "on"), (M.SYSLEN, "across")])
def test_one_launch_past_4gib(native, oracle, framing, edges):
    n = LAUNCH_LINES
    # the two line shapes, encoded once each by the oracle
    recs = []
    for x in (0, 1):
        w = LO.decode_encode_ltsv(oracle, R5, *oracle.pack([_big_line(x)]), extra=BIG_EXTRA, nthreads=1)[0]
        assert w
        recs.append(M.MERGERS[framing](w))
    r0 = len(recs[0])
    assert len(recs[1]) == r0 + 1
    # "on": records start exactly at 2^31 and 2^32; "across": at 2^31, and one record ends one byte past 2^32
    targets = (E31, E32) if edges == "on" else (E31, E32 + 1 - r0)
    extra, at = _tune(n, r0, targets)
    lens = r0 + extra
    starts = np.zeros(n + 1, np.int64)
    np.cumsum(lens, out=starts[1:])
    assert [int(starts[j]) for j in at] == list(targets)
    if edges == "across":
        assert int(starts[at[1] + 1]) == E32 + 1
    total = int(starts[-1])
    assert total > E32 + (64 << 20)
    base = len(_big_line(0))
    data, offs = _pack((_big_line(int(x)) for x in extra), n, n * base + int(extra.sum()))
    cuts = list(range(0, n, SLICE)) + [n]

    def want_digest(k):
        h = hashlib.blake2b(digest_size=16)
        for x in extra[cuts[k]:cuts[k + 1]]:
            h.update(recs[x])
        return h.digest()
    with ThreadPoolExecutor(NTHREADS) as ex:
        want = list(ex.map(want_digest, range(len(cuts) - 1)))

    dec = native.BatchDecoder(R5, max_batch_bytes=64 << 20, max_batch_lines=n + 64)
    try:
        dec.set_ltsv_extra(BIG_EXTRA)
        dec.set_output_framing(framing)
        buf, o, st, _ = dec.decode_encode_ltsv(data, offs, copy=False)
        assert len(o) == n + 1 and int(o[0]) == 0
        d = np.diff(o)
        i = _first(d < 0)
        assert i is None, f"record offsets go down at line {i}: {int(o[i])} -> {int(o[i + 1])}"
        assert int(o[-1]) == total, f"the records end at {int(o[-1])}, the oracle's at {total}"
        i = _first(d != lens)
        assert i is None, f"line {i}: record of {int(d[i])} bytes, the oracle's has {int(lens[i])}"
        assert not st.any(), f"line {_first(st != 0)}: status {int(st[st != 0][0])}"
        with ThreadPoolExecutor(NTHREADS) as ex:
            got = list(ex.map(lambda k: _digest(buf[int(o[cuts[k]]):int(o[cuts[k + 1]])]), range(len(cuts) - 1)))
        for k, (g, w) in enumerate(zip(got, want)):
            if g != w:
                for i in range(cuts[k], cuts[k + 1]):
                    assert bytes(buf[o[i]:o[i + 1]]) == recs[extra[i]], f"line {i}: record differs from the oracle's"
        assert got == want
        del buf, o, st
        # the same context, its output buffer regrown and its launch base past 4 GiB, on a small batch: the oracle's
        # records, and a fresh context's
        dec.set_ltsv_extra({})
        dec.set_output_framing(M.NONE)
        small = E.window_lines(R5)[:300]
        sd, so = oracle.pack(small)
        sbuf, soffs, sst, _ = dec.decode_encode_ltsv(sd, so)
        swant = LO.decode_encode_ltsv(oracle, R5, sd, so, nthreads=NTHREADS)
        assert [sbuf[soffs[i]:soffs[i + 1]] for i in range(len(small))] == swant
        fresh = native.BatchDecoder(R5, max_batch_bytes=1 << 20, max_batch_lines=1 << 12)
        try:
            fbuf, fo, fst, _ = fresh.decode_encode_ltsv(sd, so)
        finally:
            fresh.close()
        assert sbuf == fbuf and np.array_equal(soffs, fo) and np.array_equal(sst, fst)
    finally:
        dec.close()


# ---- spans past the segment length fields ------------------------------------------------------------------------------

BIG = (1 << 30) + (64 << 20)


def _one(native, src, line):
    dec = native.BatchDecoder(src, max_batch_bytes=BIG, max_batch_lines=64, ltsv_schema=None)
    d = np.frombuffer(line, np.uint8)
    o = np.array([0, len(line)], np.int32)
    return dec, d, o


@pytest.mark.parametrize("src", [LTSV, R5])
def test_ltsv_value_past_29_bits(native, oracle, src):
    n = (1 << 29) + 13
    if src == LTSV:  # (a TAB would end the LTSV part)
        line = b"time:1.5\thost:h\tmessage:" + b"ab:c " * (n // 5) + b"x" * (n % 5)
    else:
        line = b"<13>1 " + E.TS + b" h a p id - " + b"ab\tc:" * (n // 5) + b"x" * (n % 5)
    dec, d, o = _one(native, src, line)
    try:
        buf, offs, st, _ = dec.decode_encode_ltsv(d, o, copy=False)
        want = LO.decode_encode_ltsv(oracle, src, d, o, nthreads=1)[0]
        assert st[0] == 0 and len(want) > n
        got = buf[offs[0]:offs[1]]
        assert len(got) == len(want), f"record of {len(got)} bytes, the oracle's has {len(want)}"
        assert bytes(got) == want
    finally:
        dec.close()


def test_gelf_string_past_30_bits(native, oracle):
    n = (1 << 30) + 13
    line = b'{"host":"h","short_message":"' + b"x" * n + b'","timestamp":1.5}'
    dec, d, o = _one(native, GELF, line)
    try:
        buf, offs, st, _ = dec.decode_encode_gelf(d, o, copy=False)
        wbuf, wo = oracle.decode_encode_gelf(GELF, d, o, nthreads=1)
        assert st[0] == 0 and len(wbuf) > n
        got = buf[offs[0]:offs[1]]
        assert len(got) == len(wbuf), f"record of {len(got)} bytes, the oracle's has {len(wbuf)}"
        assert bytes(got) == wbuf
    finally:
        dec.close()


@pytest.mark.parametrize("out", ["ltsv", "gelf"])
def test_escaped_gelf_string_past_the_field_fails(native, out):
    """a string with JSON escapes is not cut into segments: one longer than the field fails the call"""
    n = (1 << 29) + 13 if out == "ltsv" else (1 << 30) + 13
    line = b'{"host":"h","short_message":"\\n' + b"x" * n + b'"}'
    dec, d, o = _one(native, GELF, line)
    try:
        call = dec.decode_encode_ltsv if out == "ltsv" else dec.decode_encode_gelf
        with pytest.raises(RuntimeError, match=re.escape("a GELF string with escapes is too long to encode")):
            call(d, o, copy=False)
        small = b'{"host":"h","short_message":"\\nm","timestamp":1}'
        buf, offs, st, _ = call(np.frombuffer(small, np.uint8), np.array([0, len(small)], np.int32))
        assert st[0] == 0 and buf  # the context still works
    finally:
        dec.close()
