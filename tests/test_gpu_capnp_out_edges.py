"""The fused Cap'n Proto encoder at its own edges, against the oracle's decoders and CapnpEncoder::encode restated
(tests/capnp_oracle.py), every message also read back by the wire-format reader, statuses against fg_decode_batch:
  - records whose segment lists end on and around the window boundaries (64, 128, 192 entries), every kind of entry
    (capnp_out_edges.KINDS) on the last entry of a window and on the first of the next, with and without
    output.capnp_extra, framed by the mergers;
  - multi-segment layouts built on purpose: pair texts that back-fill segment 0 or open segment 2, an extras list that
    opens a segment, segment tables of 3 to 6 segments; and 300 random multi-segment LTSV and GELF records;
  - GELF strings (every \\uXXXX at every offset mod 4, surrogate pairs, short escapes, raw UTF-8, newline-retry forms)
    as host, short_message, full_message, member names and member values: the unescape step of run_capnp;
  - RFC5424 lines past 64 KiB (wide rows), with the first element's pairs past byte 65535, without pairs, alone;
  - length class 63, a CTA span read from global memory, warps with a rejected line and records of 64 / 128 entries or
    four windows at every lane, records of thousands of pairs;
  - one launch whose output passes 2^32 bytes;
  - the length refusal: a GELF string whose raw span passes 2^29 bytes but whose text does not is written, a text of
    2^29 - 1 bytes is refused naming its record, and fg_set_capnp_extra refuses extras no record can hold.  GPU only."""
import ctypes as C
import hashlib
import os
import random
import re
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest

import capnp_oracle as O
import capnp_out_edges as E
import kernel_edges as KE
import ltsv_out_edges as LE
import merger_oracle as M
from flowgger_b200.native import FgEncodedOut
from test_emu_ltsv_json import RETRY
from test_gpu_encode_capnp import EDGES as CAPNP_EDGES
from test_gpu_encode_sizes import E31, E32, LAUNCH_LINES, SLICE, _digest, _first, _pack
from test_gpu_ltsv_out_edges import _bodies

pytestmark = pytest.mark.gpu
R5, LTSV, GELF, R3 = 0, 1, 2, 3
YEAR = 2026
NTHREADS = os.cpu_count() or 8
FG_E_ARG = -1


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
    """every record equals the oracle's (framed by the merger) and reads back to the oracle's Record, every status is
    fg_decode_batch's; returns the oracle's Records"""
    d, o = oracle.pack(lines)
    dec.set_capnp_extra(extra or {})
    dec.set_output_framing(framing)
    try:
        buf, offs, st, _ = dec.decode_encode_capnp(d, o)
    finally:
        dec.set_output_framing(M.NONE)
        dec.set_capnp_extra({})
    now = dec.gelf_now() if src == GELF else None
    recs = O.decode_records(oracle, src, d, o, cfg=_cfg(oracle, src), now=now, nthreads=NTHREADS)
    ex = O.extra_pairs(extra)
    for i, r in enumerate(recs):
        g = buf[offs[i]:offs[i + 1]]
        w = O.encode(r, ex) if r is not None else b""
        assert g == (M.MERGERS[framing](w) if w else b""), \
            f"record {i}: line {lines[i][:300]!r}\n got  {g[:400]!r}\n want {w[:400]!r}"
        if w:  # (the device's message is w, framed)
            assert O.read(w) == (O.as_read(r), ex)
    assert np.array_equal(st, dec.decode(d, o).status.astype(np.uint8))
    assert [r is not None for r in recs] == [s == 0 for s in st]
    return recs


# ---- segment windows --------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("framing", [M.NONE, M.SYSLEN, M.NUL])
@pytest.mark.parametrize("src", [R5, LTSV, GELF, R3])
def test_segment_windows(decs, oracle, src, framing):
    dec = decs(src)
    lines = E.window_lines(src)
    cells, totals, after = set(), set(), set()
    for extra in (None, E.EXTRA):
        recs = _check(dec, oracle, src, lines, extra, framing)
        assert all(r is not None for r in recs)
        for r in recs:
            c, t, a = E.cells(r, O.extra_pairs(extra), src)
            cells, after = cells | c, after | a
            totals.add(t)
    # every kind of entry the source emits sits on the last entry of the first and second window and on the first of
    # the second and third; windows start one entry past a whole list in segment 0 and in segment 1
    missing = {(b, k) for b in E.BOUNDARIES for k in E.KINDS[src]} - cells
    assert not missing, sorted(missing)
    assert not E.AFTER_LIST[src] - after
    if src != R3:  # an RFC3164 record has no pairs: it never reaches a second window
        assert set(E.TOTALS) <= totals


# ---- layouts over several message segments ----------------------------------------------------------------------------

def _log(r, extra, src):
    return E.model(r, extra, src)[3]


@pytest.mark.parametrize("src", [R5, LTSV, GELF])
def test_layouts(decs, oracle, src):
    dec = decs(src)
    for name, lines in E.layout_lines(src).items():
        extra = E.MANY_EXTRAS if name == "extras" else None
        ex = O.extra_pairs(extra)
        recs = _check(dec, oracle, src, lines, extra)
        assert all(r is not None for r in recs), name
        logs = [_log(r, ex, src) for r in recs]
        if name == "backfill":  # a text of a list in segment 1 has its landing pad in segment 0
            assert any(pl[0] == 0 and pl[2] is not None and ps == 1 for m in logs for ps, _, pl, _, _ in m.log)
        elif name == "segment2":  # ... and in a new segment 2
            assert any(pl[0] == 2 and ps == 1 for m in logs for ps, _, pl, _, _ in m.log)
        elif name == "extras":  # the extras list opens a new segment, behind a landing pad
            for m in logs:
                _, _, (s, _, pad), _, _ = m.log[len(m.log) - 1 - 2 * len(ex)]
                assert s == len(m.size) - 1 > 0 and pad is not None and len(m.words[s]) > 1 + 4 * len(ex)
        else:  # segment tables of an odd and an even number of entries
            nsegs = {len(m.size) for m in logs}
            assert {3, 4, 5, 6} <= nsegs if src == GELF else max(nsegs) >= 3, nsegs


@pytest.mark.parametrize("src", [LTSV, GELF])
def test_random_multi_segment_lines(decs, oracle, src):
    """the device counterpart of test_emu_capnp_out.test_random_multi_segment: 300 random records as lines"""
    rng = random.Random(7)
    dec = decs(src)
    lines = []
    for _ in range(300):
        def txt():
            return b"t" * rng.choice([0, 1, 7, 8, 100, 3000, 9000, 20000, 70000])
        n = rng.choice([0, 1, 3, 40])
        if src == LTSV:
            parts = [b"k%d:%s" % (j, txt()) if rng.random() < 0.7 else b"counter:%d" % rng.getrandbits(64) for j in range(n)]
            lines.append(LE.ltsv_line(parts, host=txt()).replace(b"message:m", b"message:" + txt()))
        else:
            mem = [b'"_k%d":"%s"' % (j, txt()) if rng.random() < 0.7 else b'"_k%d":%d' % (j, rng.getrandbits(63)) for j in range(n)]
            lines.append(b'{"host":"' + txt() + b'","short_message":"' + txt() + b'","full_message":"' + txt() +
                         b'","timestamp":1.5' + b"".join(b"," + m for m in mem) + b"}")
    extra = {"x%d" % j: "t" * rng.choice([0, 100, 9000]) for j in range(5)}
    recs = _check(dec, oracle, src, lines, extra)
    assert sum(r is not None for r in recs) >= 290
    assert max(len(_log(r, O.extra_pairs(extra), src).size) for r in recs if r is not None) >= 3


# ---- GELF strings on the device ----------------------------------------------------------------------------------------

@pytest.mark.parametrize("where", ["host", "short_message", "full_message", "key", "value"])
def test_gelf_strings(decs, oracle, where):
    dec = decs(GELF, max_batch_bytes=64 << 20, max_batch_lines=1 << 19)
    if where in ("host", "short_message", "full_message"):
        lines = [b'{"host":"h","short_message":"m","timestamp":1,"' + where.encode() + b'":"' + b + b'"}' for b in _bodies()]
        lines = [l.replace(b'"host":"h",', b"", 1) if where == "host" else l for l in lines]
        lines = [l.replace(b'"short_message":"m",', b"", 1) if where == "short_message" else l for l in lines]
    elif where == "key":
        lines = [b'{"host":"h","short_message":"m","timestamp":1,"' + b + b'":"v"}' for b in _bodies()]
        lines += [b'{"host":"h","short_message":"m","timestamp":1,"' + p + b + b'":"v"}' for p in (b"_", b"\\u005f")
                  for b in _bodies()]
    else:
        lines = [b'{"host":"h","short_message":"m","timestamp":1,"_k":"' + b + b'"}' for b in _bodies()]
    recs = _check(dec, oracle, GELF, lines)
    assert sum(r is not None for r in recs) >= 0.99 * len(lines)


def _retry_lines():
    lines = []
    for b in RETRY:
        lines += [b'{"host":"h\n","short_message":"' + b + b'","timestamp":1}',
                  b'{"host":"' + b + b'","short_message":"m","full_message":"' + b + b'","timestamp":1}',
                  b'{"host":"h","short_message":"m","timestamp":1,"_' + b + b'":"' + b + b'"}']
    return lines


def test_gelf_retry_lines(decs, oracle):
    """lines with a raw LF (the decoder's newline retry, c.mode2): pre-framed, and split from a NUL-framed stream"""
    dec = decs(GELF)
    lines = _retry_lines()
    recs = _check(dec, oracle, GELF, lines)
    assert sum(r is not None for r in recs) >= 2 * len(lines) // 3  # (the decoder rejects some `\\` + LF forms)
    d, o = oracle.pack(lines)
    pre, po, pst, _ = dec.decode_encode_capnp(d, o)
    stream = np.frombuffer(b"\0".join(lines) + b"\0", np.uint8).copy()
    buf, offs, st, _, _ = dec.split_decode_encode_capnp(stream, 1)
    assert np.array_equal(st, pst)
    for i in range(len(lines)):
        assert buf[offs[i]:offs[i + 1]] == pre[po[i]:po[i + 1]], lines[i]


# ---- wide RFC5424 rows ------------------------------------------------------------------------------------------------

def _wide(line: bytes, to: int = 70_000) -> bytes:
    """an RFC5424 line padded past 64 KiB with its message (a line without a message gets one)"""
    return line + b"p" * (to - len(line))


def test_wide_rfc5424_rows(decs, oracle):
    dec = decs(R5)
    pad = b"x" * 66_000
    lines = [_wide(l if l.endswith(b" ") else l + b" ") for l in CAPNP_EDGES["rfc5424"]]
    head = b"<13>1 " + E.TS + b" h a p id "
    lines += [
        head + b'[big@1 a="' + pad + b'" b="c\\"d" e="f"][y@2 g="h"] m',          # the first element's pairs past 65535
        head + b'[first@1 ][y@2 k="' + pad + b'"][z@3 a="b"] m',                 # the first element without pairs
        head + b'[only@1 a="b\\]c" d="' + pad + b'"] m',                          # the only element, escaped values
        head + b"[only@1 ] " + pad,                                               # the only element, no pairs
        head + b'[e@1 a="\\\\" b="\\"" c="' + pad + b'"][f@2 x="\\]"] m',
    ]
    # both sides of the switch to wide rows (lines of 65535 and 65536 bytes)
    sixteen, _ = KE.r5_sixteen_bit(7)
    wide = KE.r5_long_wide(sixteen)
    assert wide and len(wide) < len(sixteen)
    lines += sixteen
    assert len(KE.r5_long_wide(lines)) >= len(wide) + 10
    for extra in (None, {"x": "y"}):
        recs = _check(dec, oracle, R5, lines, extra)
        assert all(r is not None for r in recs)
    ids = [r["sd"][0][0] for r in recs[len(CAPNP_EDGES["rfc5424"]):len(CAPNP_EDGES["rfc5424"]) + 5]]
    assert ids == [b"big@1", b"first@1", b"only@1", b"only@1", b"e@1"]
    assert [len(recs[len(CAPNP_EDGES["rfc5424"]) + k]["sd"]) for k in (1, 2, 3)] == [3, 1, 1]
    assert [len(recs[len(CAPNP_EDGES["rfc5424"]) + k]["sd"][0][1]) for k in (1, 3)] == [0, 0]


# ---- tiles and lanes --------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("framing", [M.NONE, M.SYSLEN, M.NUL])
@pytest.mark.parametrize("src", [R5, LTSV, GELF, R3])
def test_tiles_and_lanes(decs, oracle, src, framing):
    dec = decs(src)
    rng = np.random.default_rng(40 + src)
    _check(dec, oracle, src, LE.long_lines(src, rng), E.EXTRA, framing)
    span = LE.span_lines(src, rng)
    _, o = oracle.pack(span)
    assert int(o[256 * 5] - o[256 * 4]) > 4 * 32768  # above every encoder tile
    _check(dec, oracle, src, span, None, framing)
    recs = _check(dec, oracle, src, E.lane_lines(src, rng), None, framing)
    assert sum(r is None for r in recs) == 32 * (2 if src == R3 else 3)


# pairs per line: several thousand, within what each decoder accepts on one line
MANY = {R5: 4000, LTSV: 4000, GELF: 4000}


@pytest.mark.parametrize("src", [R5, LTSV, GELF])
def test_thousands_of_pairs(decs, oracle, src):
    """one lane runs hundreds of windows: a record of thousands of pairs, beside short ones in the same warp"""
    dec = decs(src)
    n = MANY[src]
    big = E._line(src, [E._PAIRS[src][0](k) for k in range(n)], 0)
    lines = [E._line(src, [E._PAIRS[src][0](0)], 0)] * 31
    lines = lines[:13] + [big] + lines[13:]
    recs = _check(dec, oracle, src, lines, E.EXTRA)
    r = recs[13]
    assert r is not None and len(r["sd"][0][1]) == n
    assert len(E.segments(r, O.extra_pairs(E.EXTRA), src)) > 100 * E.WINDOW


# ---- one launch past 2^32 bytes of output -----------------------------------------------------------------------------

# A ~9.8 KB output.capnp_extra value makes every record of a ~41-byte RFC5424 line a two-segment message of ~10 KB: the
# 512 Ki lines of one launch (the default chunk_lines) pass 4 GiB of output from 21 MB of input.  A capnp record grows
# in whole words: eight more fraction digits of the timestamp (the same Record.ts) are one more word of full_msg only,
# which places records exactly (_tune_bytes, in steps of 8 bytes).  Under syslen a record of five length digits is framed
# to an odd length, so a record can end on any byte.
BIG_EXTRA = {"e": "x" * 9800}


def _big_line(extra: int) -> bytes:
    return b"<13>1 2015-08-05T15:53:45.5" + b"0" * (8 * extra) + b"Z h a p id - m"


@pytest.mark.parametrize("framing,edges", [(M.NONE, "on"), (M.SYSLEN, "across")])
def test_one_launch_past_4gib(native, oracle, framing, edges):
    n = LAUNCH_LINES
    ex = O.extra_pairs(BIG_EXTRA)
    recs = []
    for x in (0, 1):
        r = O.decode_records(oracle, R5, *oracle.pack([_big_line(x)]), nthreads=1)[0]
        recs.append(M.MERGERS[framing](O.encode(r, ex)))
    assert len(_log(r, ex, R5).size) == 2
    # the unframed records are whole words; syslen puts a decimal prefix of the same length before both
    r0 = len(recs[0])
    step = len(recs[1]) - r0
    assert step == 8 and (framing != M.NONE or r0 % 8 == 0)
    # "on": records start exactly at 2^31 and 2^32; "across": at 2^31, and one record ends one byte past 2^32
    targets = (E31, E32) if edges == "on" else (E31, E32 + 1 - r0)
    extra, at = _tune_bytes(n, r0, step, targets)
    lens = r0 + step * extra
    starts = np.zeros(n + 1, np.int64)
    np.cumsum(lens, out=starts[1:])
    assert [int(starts[j]) for j in at] == list(targets)
    if edges == "across":
        assert int(starts[at[1] + 1]) == E32 + 1
    total = int(starts[-1])
    assert total > E32 + (64 << 20)
    base = len(_big_line(0))
    data, offs = _pack((_big_line(int(x)) for x in extra), n, n * base + 8 * int(extra.sum()))
    cuts = list(range(0, n, SLICE)) + [n]

    def want_digest(k):
        h = hashlib.blake2b(digest_size=16)
        for x in extra[cuts[k]:cuts[k + 1]]:
            h.update(recs[x])
        return h.digest()
    with ThreadPoolExecutor(NTHREADS) as ex_:
        want = list(ex_.map(want_digest, range(len(cuts) - 1)))

    dec = native.BatchDecoder(R5, max_batch_bytes=64 << 20, max_batch_lines=n + 64)
    try:
        dec.set_capnp_extra(BIG_EXTRA)
        dec.set_output_framing(framing)
        buf, o, st, _ = dec.decode_encode_capnp(data, offs, copy=False)
        assert len(o) == n + 1 and int(o[0]) == 0
        d = np.diff(o)
        i = _first(d < 0)
        assert i is None, f"record offsets go down at line {i}: {int(o[i])} -> {int(o[i + 1])}"
        assert int(o[-1]) == total, f"the records end at {int(o[-1])}, the oracle's at {total}"
        i = _first(d != lens)
        assert i is None, f"line {i}: record of {int(d[i])} bytes, the oracle's has {int(lens[i])}"
        assert not st.any(), f"line {_first(st != 0)}: status {int(st[st != 0][0])}"
        with ThreadPoolExecutor(NTHREADS) as ex_:
            got = list(ex_.map(lambda k: _digest(buf[int(o[cuts[k]]):int(o[cuts[k + 1]])]), range(len(cuts) - 1)))
        for k, (g, w) in enumerate(zip(got, want)):
            if g != w:
                for i in range(cuts[k], cuts[k + 1]):
                    assert bytes(buf[o[i]:o[i + 1]]) == recs[extra[i]], f"line {i}: record differs from the oracle's"
        assert got == want
        del buf, o, st
        # the same context, its output buffer regrown and its launch base past 4 GiB, on a small batch: the oracle's
        # records, and a fresh context's
        dec.set_capnp_extra({})
        dec.set_output_framing(M.NONE)
        small = E.window_lines(R5)[:300]
        sd, so = oracle.pack(small)
        sbuf, soffs, sst, _ = dec.decode_encode_capnp(sd, so)
        swant = O.decode_encode_capnp(oracle, R5, sd, so, nthreads=NTHREADS)
        assert [sbuf[soffs[i]:soffs[i + 1]] for i in range(len(small))] == swant
        fresh = native.BatchDecoder(R5, max_batch_bytes=1 << 20, max_batch_lines=1 << 12)
        try:
            fbuf, fo, fst, _ = fresh.decode_encode_capnp(sd, so)
        finally:
            fresh.close()
        assert sbuf == fbuf and np.array_equal(soffs, fo) and np.array_equal(sst, fst)
    finally:
        dec.close()


def _tune_bytes(n, r0, step, targets):
    """_tune for records of r0 + step * extra[i] bytes: one record starts exactly at each offset of `targets`"""
    extra = np.zeros(n, np.int64)
    j0, s0, lines = 0, 0, []
    for s in targets:
        j = j0 + (s - s0) // r0
        rest = (s - s0) - (j - j0) * r0
        for _ in range(step):  # one line fewer before the target leaves r0 more bytes to spread
            if rest % step == 0:
                break
            j -= 1
            rest += r0
        assert rest % step == 0, f"no record can start at {s}"
        need = rest // step
        assert j < n and need <= j - j0, (s, need, j - j0)
        extra[j0:j0 + need] = 1
        lines.append(j)
        j0, s0 = j, s
    return extra, lines


# ---- the length refusal -----------------------------------------------------------------------------------------------

CAP = 1 << 29
HEAVY = (CAP + (64 << 20))


def _escaped(k: int) -> bytes:
    """1,000 \\u0041 escapes then plain bytes: a text of k bytes from a span of k + 5,000"""
    return b"\\u0041" * 1000 + b"x" * (k - 1000)


def _one_line(native, line):
    dec = native.BatchDecoder(GELF, max_batch_bytes=HEAVY, max_batch_lines=64)
    return dec, np.frombuffer(line, np.uint8), np.array([0, len(line)], np.int32)


def test_escaped_string_past_29_bits(native):
    """a GELF short_message whose raw span passes 2^29 bytes but whose text is 2^29 - 2 bytes is written; one byte more
    is refused.  (The same string as a member value is not run here: one thread walks its unescape three times in the
    write pass, about 1.1 us per byte on an H100, some ten minutes at this length.)"""
    for k, ok in ((CAP - 2, True), (CAP - 1, False)):
        s = _escaped(k)
        assert len(s) > CAP
        dec, d, o = _one_line(native, b'{"host":"h","short_message":"' + s + b'","timestamp":1.5}')
        try:
            if not ok:
                out = FgEncodedOut()
                rc = dec.L.fg_decode_encode_capnp(dec.ctx, GELF, d.ctypes.data, o.ctypes.data, 1, C.byref(out))
                assert rc == FG_E_ARG
                assert b"record 0: a text of 2^29 - 1 bytes" in dec.L.fg_last_error(dec.ctx)
                continue
            buf, offs, st, _ = dec.decode_encode_capnp(d, o, copy=False)
            assert st[0] == 0
            rec, extra = O.read(bytes(buf[offs[0]:offs[1]]))
            assert extra == [] and rec["host"] == b"h" and rec["ts_bits"] == 0x3FF8000000000000 and rec["sd"] is None
            assert rec["msg"] == b"A" * 1000 + b"x" * (k - 1000)
        finally:
            dec.close()


@pytest.mark.parametrize("split", [False, True])
def test_refusal_names_the_record(native, split):
    """a text of 2^29 - 1 bytes in a later parse step (chunk_lines = 1000), after empty lines: the error names it"""
    head = b"<13>1 2015-08-05T15:53:45Z h a p m - "
    long_line = head + b"m" * (CAP - 1 - len(head))  # full_msg is the whole line
    ok = b"<13>1 2015-08-05T15:53:45Z h a p m - ok"
    at = 2500
    lines = [ok] * (at - 3) + [b""] * 3 + [long_line] + [ok] * 700
    dec = native.BatchDecoder(R5, chunk_lines=1000, max_batch_bytes=CAP + (16 << 20), max_batch_lines=1 << 13)
    try:
        out = FgEncodedOut()
        if split:
            stream = np.frombuffer(b"\n".join(lines) + b"\n", np.uint8)
            lo = C.POINTER(C.c_int32)()
            rc = dec.L.fg_split_decode_encode_capnp(dec.ctx, R5, 0, stream.ctypes.data, len(stream), C.byref(out), C.byref(lo))
        else:
            d, o = _pack(lines, len(lines), sum(map(len, lines)))
            rc = dec.L.fg_decode_encode_capnp(dec.ctx, R5, d.ctypes.data, o.ctypes.data, len(lines), C.byref(out))
        assert rc == FG_E_ARG
        assert re.search(rb"record (\d+):", dec.L.fg_last_error(dec.ctx)).group(1) == b"%d" % at
        # the context still works
        sd, so = _pack([ok] * 3, 3, 3 * len(ok))
        buf, offs, st, _ = dec.decode_encode_capnp(sd, so)
        assert list(st) == [0, 0, 0] and O.read(buf[offs[2]:offs[3]])[0]["msg"] == b"ok"
    finally:
        dec.close()


def test_extra_limits(decs, oracle):
    """fg_set_capnp_extra refuses a value of 2^29 - 1 bytes and extras of more than 2^31 - 1 bytes in all, and keeps the
    extras in use; set calls only"""
    dec = decs(R5)
    L = dec.L
    dec.set_capnp_extra({"k": "v"})
    big = b"v" * (CAP - 1)

    def call(keys, vals):
        return L.fg_set_capnp_extra(dec.ctx, len(keys), (C.c_char_p * len(keys))(*keys), (C.c_char_p * len(vals))(*vals))
    assert call([b"a"], [big]) == FG_E_ARG
    assert b"2^29 - 1" in L.fg_last_error(dec.ctx)
    assert call([big], [b"a"]) == FG_E_ARG
    just = big[:-1]  # 2^29 - 2 bytes each: five of them are more than 2^31 - 1 bytes
    assert call([b"a%d" % k for k in range(5)], [just] * 5) == FG_E_ARG
    assert b"2^31 - 1" in L.fg_last_error(dec.ctx)
    lines = [b"<13>1 2015-08-05T15:53:45Z h a p m - m"]
    d, o = oracle.pack(lines)
    buf, _, st, _ = dec.decode_encode_capnp(d, o)
    assert st[0] == 0 and O.read(buf)[1] == [(b"k", b"v")]  # unchanged by the refused calls
    dec.set_capnp_extra({})
