"""The front end every raw-stream call shares (framing at '\\n' or NUL, the from_utf8 check of each record, the 64 MiB
chunk pipeline) against pysplit and Python's strict UTF-8 decoder, at its own edges: every short byte sequence,
sequences next to delimiters and to each other, events at every offset around a chunk seam, records longer than a
chunk, stream lengths around chunk multiples, and record and byte counts at a context's capacity.  GPU only."""
import functools
import os

import numpy as np
import pytest

import split_edges as S

pytestmark = pytest.mark.gpu

R5 = 0  # FMT_RFC5424
NTHREADS = os.cpu_count() or 4
FRAMINGS = {"line": 0, "nul": 1}
ENCODERS = ("gelf", "ltsv", "capnp", "passthrough")
CAP = 4096  # max_batch_lines of the capacity context: a multiple of 64, so not rounded
MORE_LINES = "stream has more lines than max_batch_lines"
MORE_BYTES = "stream has more bytes than max_batch_bytes"


@pytest.fixture(scope="module")
def big(native):
    dec = native.BatchDecoder(R5, max_batch_bytes=256 << 20, max_batch_lines=3 << 20)
    yield dec
    dec.close()


@pytest.fixture(scope="module")
def cap(native):
    dec = native.BatchDecoder(R5, max_batch_bytes=128 << 20, max_batch_lines=CAP)
    yield dec
    dec.close()


def _arr(stream) -> np.ndarray:
    return np.frombuffer(stream, np.uint8) if isinstance(stream, bytes) else stream


def _line_offsets(res) -> np.ndarray:
    return np.ctypeslib.as_array(res.raw.line_offsets, shape=(res.n + 1,)).copy()


def _want_dumps(oracle, lines: list[bytes], valid: list[bool]) -> list[bytes]:
    """per record: the oracle's decode of the stripped record, or the UTF-8 error where Python's decoder refuses it"""
    d, o = _pack([l for l, v in zip(lines, valid) if v])
    obuf, oo = oracle.decode_dump(R5, d, o, nthreads=NTHREADS)
    want, k = [], 0
    for v in valid:
        want.append(obuf[oo[k]:oo[k + 1]] if v else S.UTF8_ERROR_DUMP)
        k += v
    return want


def _compare(dec, a: np.ndarray, framing: str, offs: np.ndarray, want: bytes, want_lens: np.ndarray, lines) -> None:
    """fg_split_decode_framed on `a`: the record starts `offs` and the dumps `want` (record i: want_lens[i] bytes)"""
    buf, bo, lo, _ = dec.split_dump(a, FRAMINGS[framing])
    assert np.array_equal(lo, offs), (len(lo), len(offs), np.flatnonzero(lo[:len(offs)] != offs[:len(lo)])[:5])
    if buf != want or not np.array_equal(np.diff(bo), want_lens):
        wo = np.concatenate([[0], np.cumsum(want_lens)])
        bad = next(i for i in range(len(want_lens)) if buf[bo[i]:bo[i + 1]] != want[wo[i]:wo[i + 1]])
        raise AssertionError(f"record {bad} at {offs[bad]}: {lines(bad)[-60:]!r}\n"
                             f" got  {buf[bo[bad]:bo[bad + 1]][:300]!r}\n want {want[wo[bad]:wo[bad + 1]][:300]!r}")


def check_dumps(dec, oracle, stream, framing: str) -> list[bool]:
    """fg_split_decode_framed against pysplit's record starts and, record by record, the oracle's decode of the stripped
    record or the UTF-8 error exactly where Python's decoder refuses the record.  Returns the validity flags."""
    a = _arr(stream)
    offs, lines, valid = S.expect(a.tobytes(), S.DELIMS[framing])
    want = _want_dumps(oracle, lines, valid)
    _compare(dec, a, framing, offs, b"".join(want), np.array([len(w) for w in want]), lines.__getitem__)
    return valid


def _pack(lines: list[bytes]) -> tuple[np.ndarray, np.ndarray]:
    offs = np.zeros(len(lines) + 1, np.int32)
    np.cumsum([len(l) for l in lines], out=offs[1:])
    return np.frombuffer(b"".join(lines) + b"\0", np.uint8)[:int(offs[-1])].copy(), offs


# ---- UTF-8 ------------------------------------------------------------------------------------------------------------


@pytest.mark.parametrize("batch", range(S.EXHAUSTIVE_BATCHES))
@pytest.mark.parametrize("framing", FRAMINGS)
def test_utf8_exhaustive(big, framing, batch):
    """every short sequence in a record of its own, about 2 M records per call: status FG_ES_INVALID_UTF8 exactly where
    Python's strict decoder refuses the record"""
    delim = S.DELIMS[framing]
    stream, at, ln = S.utf8_exhaustive_batch(delim, batch)
    starts, valid = S.fast_expect(stream, delim)
    res = big.split_decode(_arr(stream), FRAMINGS[framing])
    assert np.array_equal(_line_offsets(res), starts)
    flagged = res.status == S.INVALID_UTF8
    wrong = np.flatnonzero(flagged == valid)
    assert len(wrong) == 0, (len(wrong), [(stream[at[i]:at[i] + ln[i]].hex(), bool(valid[i])) for i in wrong[:10]])


@pytest.mark.parametrize("framing", FRAMINGS)
def test_utf8_in_context(big, oracle, framing):
    """stray continuation bytes, a continuation byte right after a delimiter, a lead right before one (and before
    "\\r\\n"), two invalid sequences in a record, invalid and valid records sharing a 16-byte window"""
    stream, _ = S.utf8_in_context(S.DELIMS[framing])
    valid = check_dumps(big, oracle, stream, framing)
    assert 0 < sum(valid) < len(valid)


# ---- the chunk pipeline -----------------------------------------------------------------------------------------------


@functools.lru_cache(maxsize=2)
def _seam_base_expected(oracle, framing: str):
    """the base stream of chunk_seam framed by pysplit, split around the record that spans the seam: (record starts,
    that record's index, the dumps before it and their lengths, the dumps after it and their lengths)"""
    offs, lines, valid = S.expect(S.seam_base(S.DELIMS[framing]).tobytes(), S.DELIMS[framing])
    assert all(valid)
    r = int(np.searchsorted(offs, S.CHUNK, side="right")) - 1
    want = _want_dumps(oracle, lines, valid)
    lens = np.array([len(w) for w in want])
    return offs, r, b"".join(want[:r]), lens[:r], b"".join(want[r + 1:]), lens[r + 1:]


@pytest.mark.parametrize("kind", S.SEAM_EVENTS)
@pytest.mark.parametrize("framing", FRAMINGS)
def test_chunk_seam(big, oracle, framing, kind):
    """one event at every offset from 20 bytes before the first 64 MiB seam to 19 after it: the lag window of the
    validation (c1 - 16) and the 3-byte read-ahead of a lead both cross the seam.  An event only changes the record
    that spans the seam, which starts after a delimiter and ends with one far from the event, so pysplit frames that
    record alone and the rest of the stream once."""
    delim = S.DELIMS[framing]
    refused = kind in ("stray", "lead", "overlong", "surrogate")
    offs, r, pre, pre_lens, post, post_lens = _seam_base_expected(oracle, framing)
    lo, hi = int(offs[r]), int(offs[r + 1])
    for where in S.SEAM_WHERE:
        a, _ = S.chunk_seam(delim, where, kind)
        loffs, lines, valid = S.expect(a[lo:hi].tobytes(), delim)
        assert valid.count(False) == refused and len(lines) == 1 + kind.endswith("delim"), where
        want = _want_dumps(oracle, lines, valid)
        _compare(big, a, framing, np.concatenate([offs[:r], lo + loffs[:-1], offs[r + 1:]]),
                 pre + b"".join(want) + post, np.concatenate([pre_lens, [len(w) for w in want], post_lens]),
                 lambda i: lines[i - r] if r <= i < r + len(lines) else b"(a record of the base stream)")


@pytest.mark.parametrize("framing", FRAMINGS)
def test_long_records_and_stream_lengths(big, oracle, framing):
    """records of 64 MiB + 100 bytes and of 130 MiB (a middle chunk without a delimiter, with characters across both
    seams, with an invalid byte), and streams of k * 64 MiB + {-1, 0, 1, 15, 16, 17} bytes, terminated or not"""
    for label, stream in S.long_records(S.DELIMS[framing]):
        valid = check_dumps(big, oracle, stream, framing)
        assert all(valid) == (label != "130M-invalid"), label


# ---- capacity ---------------------------------------------------------------------------------------------------------


def _split_calls(dec, a: np.ndarray, framing: int, d: np.ndarray, o: np.ndarray):
    """(name, raw-stream call, check against the pre-framed call on the stripped records) for the six raw-stream calls;
    fg_split_decode frames at '\\n' only"""
    def dump():
        buf, bo, lo, _ = dec.split_dump(a, framing)
        pre = dec.decode(d, o)
        pbuf, pbo = dec.dump(pre, d, o)
        return lo, (buf == pbuf and np.array_equal(bo, pbo))

    def split_decode():
        res = dec.split_decode(a)
        lo, st = _line_offsets(res), res.status.copy()
        return lo, np.array_equal(st, dec.decode(d, o).status)

    def fused(enc):
        def run():
            buf, offs, st, lo, _ = getattr(dec, f"split_decode_encode_{enc}")(a, framing)
            pbuf, poffs, pst, _ = getattr(dec, f"decode_encode_{enc}")(d, o)
            return lo, (buf == pbuf and np.array_equal(offs, poffs) and np.array_equal(st, pst))
        return run

    calls = [("fg_split_decode_framed", dump)] + ([("fg_split_decode", split_decode)] if framing == 0 else [])
    return calls + [(f"fg_split_decode_encode_{e}", fused(e)) for e in ENCODERS]


@pytest.mark.parametrize("framing", FRAMINGS)
def test_capacity_lines(cap, framing):
    """max_batch_lines - 1, max_batch_lines and max_batch_lines + 1 records, terminated or not, through every raw-stream
    call: refused exactly when there are more records than max_batch_lines, the context usable after a refusal, and an
    accepted stream decoded as the pre-framed call decodes its records"""
    delim = S.DELIMS[framing]
    streams = list(S.capacity_streams(CAP, delim))
    for label, stream, n in streams + streams[:1]:  # the first stream again, after the refusals
        offs, lines, valid = S.expect(stream, delim)
        assert len(offs) - 1 == n and all(valid)
        d, o = _pack(lines)
        for name, call in _split_calls(cap, _arr(stream), FRAMINGS[framing], d, o):
            if n > CAP:
                with pytest.raises(RuntimeError, match=MORE_LINES):
                    call()
                continue
            lo, same = call()
            assert np.array_equal(lo, offs), (label, name)
            assert same, (label, name)


def test_block_splitter_exact_fit_is_one_call(native, cap):
    """BatchingLineSplitter over exactly max_batch_lines terminated records decodes them in one device call: it launches
    what one fg_split_decode of the same records does, not a refused call and two halves"""
    text = next(s for label, s, _ in S.capacity_streams(CAP, b"\n") if label == f"{CAP}-term")
    deltas = []
    for _ in range(2):  # the second call: tables already sized for these records
        n0 = cap.kernel_launches()
        cap.split_decode(_arr(text[:-1]))  # the same records, the last one unterminated
        deltas.append(cap.kernel_launches() - n0)
    n0 = cap.kernel_launches()
    _, err, _ = native.splitter_run(cap, text, max_lines=CAP, max_bytes=16 << 20)
    assert err == b""
    assert cap.kernel_launches() - n0 == deltas[-1]


def test_capacity_bytes_exact_fit(native):
    """a stream of exactly max_batch_bytes is accepted, one byte more is refused, and the context stays usable"""
    nbytes = (3 << 20) + 37
    dec = native.BatchDecoder(R5, max_batch_bytes=nbytes, max_batch_lines=1 << 16)
    try:
        rng = np.random.default_rng(21)
        a = np.empty(nbytes + 1, np.uint8)
        S.fill_records(a[:nbytes], S.records_layout(nbytes, rng, 100, 2000), b"\n", rng)
        a[nbytes] = ord("x")
        for framing in FRAMINGS.values():
            delim = b"\0" if framing else b"\n"
            b = a.copy()
            b[b == ord("\n")] = delim[0]
            for _ in range(2):
                res = dec.split_decode(b[:nbytes], framing)
                assert np.array_equal(_line_offsets(res), S.record_starts(b[:nbytes], delim))
                assert (res.status == 0).all()
                with pytest.raises(RuntimeError, match=MORE_BYTES):
                    dec.split_decode(b, framing)
    finally:
        dec.close()


def test_capacity_bytes_clamped_to_int32_offsets(native):
    """max_batch_bytes = 2^31 is clamped to 0x7FFFFFC0 for int32 offsets: a stream of exactly that length, of records
    of about 1 KiB, frames at numpy's delimiter positions up to an end offset near 2^31 and decodes as the pre-framed
    call decodes its records; one byte more is refused"""
    limit = 0x7FFFFFC0
    dec = native.BatchDecoder(R5, max_batch_bytes=1 << 31, max_batch_lines=3 << 20)
    try:
        rng = np.random.default_rng(31)
        a = np.empty(limit + 1, np.uint8)
        S.fill_records(a[:limit], S.records_layout(limit, rng, 900, 1150), b"\n", rng)
        a[limit] = ord("x")
        starts = S.record_starts(a[:limit], b"\n")
        res = dec.split_decode(a[:limit])
        lo, st = _line_offsets(res), res.status.copy()
        assert np.array_equal(lo, starts) and int(lo[-1]) == limit and len(lo) > 2_000_000
        d = a[:limit][a[:limit] != ord("\n")]  # the records without their terminators
        o = (starts - np.arange(len(starts))).astype(np.int32)
        assert np.array_equal(st, dec.decode(d, o).status) and (st == 0).all()
        with pytest.raises(RuntimeError, match=MORE_BYTES):
            dec.split_decode(a)
    finally:
        dec.close()
