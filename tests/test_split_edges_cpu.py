"""The stream builders of split_edges.py put each probe where they claim, and the numpy restatement of the references
that the exhaustive streams use agrees with pysplit record by record.  No GPU."""
import numpy as np
import pytest

import split_edges as S

DELIMS = list(S.DELIMS.values())
IDS = list(S.DELIMS)


@pytest.mark.parametrize("delim", DELIMS, ids=IDS)
def test_exhaustive_candidates_cover_the_claimed_sets(delim):
    cand, clen = S.exhaustive_candidates(delim)
    assert len(clen) == S.EXHAUSTIVE_COUNT == 128 * 255 * 255 + 5 * 255 * 255 * 7 + 5 * 255 * 4 * 255 + 128 + 128 * 255
    assert not (cand[np.arange(4)[None, :] < clen[:, None]] == delim[0]).any()
    three = cand[clen == 3]
    assert len(np.unique(three[:, 0].astype(np.int64) << 16 | three[:, 1].astype(np.int64) << 8 | three[:, 2])) == 128 * 255 * 255
    four = cand[clen == 4]
    assert set(four[:, 0]) == set(range(0xF0, 0xF5))
    assert set(four[:, 3]) == set(range(256)) - {delim[0]} and set(four[:, 2]) == set(range(256)) - {delim[0]}
    for b in (0xC0, 0xC1, 0xF5, 0xFF):  # C0 / C1 followed by every byte, F5..FF leads
        assert ((clen == 2) & (cand[:, 0] == b)).sum() == 255


@pytest.mark.parametrize("delim", DELIMS, ids=IDS)
def test_exhaustive_streams_place_every_candidate(delim):
    cand, clen = S.exhaustive_candidates(delim)
    r0 = 0
    for stream, at, ln in S.utf8_exhaustive(delim):
        r = np.arange(r0, r0 + len(at))
        a = np.frombuffer(stream, np.uint8)
        starts = S.record_starts(stream, delim)
        assert len(starts) - 1 == len(at) and a[-1] == delim[0]  # one record per candidate, all terminated
        assert (starts[:-1] <= at).all() and (at + ln < starts[1:]).all()
        assert np.array_equal(at % 16, r % 16)
        assert np.array_equal(ln, clen[r])
        for j in range(4):
            m = ln > j
            assert np.array_equal(a[at[m] + j], cand[r[m], j])
        suffix = r % 5 == 0
        cr = (r % 7 == 0) & (delim == b"\n")
        assert np.array_equal(starts[1:] - at - ln, 1 + suffix + cr)
        assert (a[(at + ln)[suffix]] == ord("a")).all() and (a[starts[1:][cr] - 2] == ord("\r")).all()
        r0 += len(at)
    assert r0 == len(clen)


@pytest.mark.parametrize("delim", DELIMS, ids=IDS)
def test_fast_expect_equals_pysplit_on_every_candidate(delim):
    """the numpy verdicts of the exhaustive streams equal pysplit's, which are bytes.decode's, for every 1-, 2-, 3- and
    4-byte candidate; the strict decoder refuses a share the Unicode tables predict"""
    invalid = 0
    for stream, at, ln in S.utf8_exhaustive(delim):
        starts, valid = S.fast_expect(stream, delim)
        offs, _, v = S.expect(stream, delim)
        assert np.array_equal(starts, offs)
        assert np.array_equal(valid, np.asarray(v, bool))
        invalid += int((~valid).sum())
    # Table 3-7 counted: a lead C2..DF + a continuation byte + ASCII (the delimiter excluded); E0, ED and E1..EC, EE, EF
    # with their second-byte ranges (32, 32, 64 each) + a continuation byte; F0, F1..F3, F4 with their second-byte ranges
    # (48, 64 each, 16) + continuation bytes, of which FOUR_B3 holds 4 and FOUR_B2 2
    cont, ascii_, second3, second4 = 64, 127, 32 + 32 + 14 * 64, 48 + 3 * 64 + 16
    valid = 30 * cont * ascii_ + second3 * cont + second4 * cont * 4 + second4 * 2 * cont + 30 * cont
    assert len(S.exhaustive_candidates(delim)[1]) - invalid == valid


def test_fast_expect_on_every_two_byte_string():
    """bytes.decode against fast_expect for every b0 b1, in records ended by the delimiter and by end of stream"""
    for delim in DELIMS:
        bs = [bytes([a, b]) for a in range(256) for b in range(256) if delim[0] not in (a, b)]
        stream = delim.join(bs)
        starts, valid = S.fast_expect(stream, delim)
        assert len(starts) - 1 == len(bs)
        want = []
        for b in bs:
            try:
                b.decode("utf-8")
                want.append(True)
            except UnicodeDecodeError:
                want.append(False)
        assert np.array_equal(valid, want)


@pytest.mark.parametrize("delim", DELIMS, ids=IDS)
def test_in_context_probes(delim):
    stream, probes = S.utf8_in_context(delim)
    offs, lines, valid = S.expect(stream, delim)
    starts, fast = S.fast_expect(stream, delim)
    assert np.array_equal(starts, offs) and np.array_equal(fast, valid)
    for name in ("stray1", "stray4", "first", "last", "two", "window"):
        at = {p % 16 for n, p in probes if n == name}
        assert at == set(range(16)), name
    a = np.frombuffer(stream, np.uint8)
    # the short records that share a 16-byte span, by their first byte: (records, validity)
    windows = {0xFF: (2, [False, False]), ord("a"): (3, [False, True, False]), 0xE6: (3, [True, False, True])}
    for name, p in probes:
        if name == "first":
            assert a[p - 1] == delim[0] and a[p] == 0x80
        if name == "window":
            rec = np.searchsorted(offs, p, side="right") - 1
            k, want = windows[a[p]]
            assert offs[rec + k] <= p + 16 and valid[rec:rec + k] == want
    assert 0 < sum(valid) < len(valid)


@pytest.mark.parametrize("delim", DELIMS, ids=IDS)
def test_chunk_seam_events(delim):
    base = S.seam_base(delim)
    assert len(base) == S.CHUNK + (64 << 10)
    offs, lines, valid = S.expect(base.tobytes(), delim)
    assert all(valid) and np.array_equal(offs, S.record_starts(base, delim))
    seam_rec = np.searchsorted(offs, S.CHUNK, side="right") - 1
    assert offs[seam_rec] < S.CHUNK - S.SEAM_QUIET and offs[seam_rec + 1] > S.CHUNK + S.SEAM_QUIET
    for kind in S.SEAM_EVENTS:
        e = S.seam_event(delim, kind)
        for where in (min(S.SEAM_WHERE), -3, -1, 0, max(S.SEAM_WHERE)):
            stream, at = S.chunk_seam(delim, where, kind)
            assert at == S.CHUNK + where and stream[at:at + len(e)].tobytes() == e
            assert set(np.flatnonzero(stream != base)) <= set(range(at, at + len(e)))
    # the read-ahead and the lag window are both inside the offsets: a 4-byte lead 3 bytes before the seam, and the first
    # byte validated with the next chunk (c1 - 16)
    assert min(S.SEAM_WHERE) < -S.LAG and max(S.SEAM_WHERE) > 3


@pytest.mark.parametrize("delim", DELIMS, ids=IDS)
def test_long_records_and_lengths(delim):
    seen = set()
    for label, stream in S.long_records(delim):
        starts = S.record_starts(stream, delim)
        ends_chunk = set((starts[1:] - 1) // S.CHUNK)  # the chunk in which each record ends
        term = stream[-1] == delim[0]
        if label.startswith(("64M", "130M")):
            assert term and len(starts) == 4
            long_len = int(starts[2] - starts[1])
            assert long_len == {"64M+100": S.CHUNK + 100}.get(label, 130 << 20)
            if label.startswith("130M"):
                assert ends_chunk == {0, 2}  # the middle chunk holds no delimiter
        else:
            k, rest = label.split("x64M")
            d, kind = rest.rsplit("-", 1)
            assert len(stream) == int(k) * S.CHUNK + int(d) and term == (kind == "term")
            assert ends_chunk == set(range(-(-len(stream) // S.CHUNK)))
            if int(k) == 1 and int(d) == 1 and term:  # the last chunk is the delimiter alone
                assert len(stream) == S.CHUNK + 1 and stream[S.CHUNK] == delim[0] and stream[S.CHUNK - 1] != delim[0]
                seen.add("delimiter alone")
        offs, _, valid = S.expect(stream.tobytes(), delim)
        assert np.array_equal(offs, starts)
        assert all(valid) == (label != "130M-invalid")
    assert seen == {"delimiter alone"}


def split_refuses(stream: bytes, max_lines: int, delim: bytes) -> bool:
    """scan_segments_kernel's capacity rule, chunk by chunk: a chunk that is not the last is refused when its delimiters
    leave no room for the record open after it; the last chunk counts an unterminated last record only"""
    a = np.frombuffer(stream, np.uint8)
    chunks = max(1, -(-len(a) // S.CHUNK))
    for k in range(chunks):
        newlines = int((a[:min(len(a), (k + 1) * S.CHUNK)] == delim[0]).sum())
        last = k == chunks - 1
        tail = last and len(a) > 0 and a[-1] != delim[0]
        if newlines + (tail if last else 1) > max_lines:
            return True
    return False


@pytest.mark.parametrize("delim", DELIMS, ids=IDS)
@pytest.mark.parametrize("max_lines", [64, 4096])
def test_capacity_rule(delim, max_lines):
    labels = []
    for label, stream, n in S.capacity_streams(max_lines, delim):
        offs, _, valid = S.expect(stream, delim)
        assert len(offs) - 1 == n and all(valid)
        assert split_refuses(stream, max_lines, delim) == (n > max_lines), label
        labels.append(label)
        if "long" in label:  # the last delimiter falls in the second chunk
            assert stream[-1] == delim[0] and (len(stream) - 1) // S.CHUNK == 1
    assert labels == [f"{n}-{t}" for n in (max_lines - 1, max_lines, max_lines + 1) for t in ("term", "open")] + [f"{max_lines}-long-term"]
