"""The fused GELF encoder (fg_decode_encode_gelf, fg_split_decode_encode_gelf) at the output sizes where 32-bit and
31-bit arithmetic breaks, against the oracle (oracle decoder -> Record -> oracle/encoder.cpp):
  - one encoder launch whose output passes 2^32 bytes, with record boundaries placed exactly on 2^31 and 2^32 or one byte
    across them (RFC5424 and RFC3164 sources, escape-heavy lines), and with realistic generated lines;
  - bench.py's workloads, whole, over many launches (RFC5424 past 2^32, RFC3164 past 2^31), framed and raw;
  - the context after such calls, on a small batch.
A single record larger than 4 GiB is not run here: one GPU thread emits a record, and its byte loop over a record past
4 GiB does not finish within nine minutes.
Host memory stays bounded: the device result is taken as views of the pinned buffers, and the oracle runs over slices of
SLICE lines, whose record lengths are kept and whose bytes are kept as a digest.  Every check first asserts what a wrap
of the record offsets breaks (offsets never go down, the last one is the sum of the oracle's record lengths), then the
record lengths, the statuses and the bytes.  GPU only."""
import hashlib
import os
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest

import vectors as V

pytestmark = pytest.mark.gpu
R5, R3 = 0, 3
YEAR = 2026  # RFC3164: the year of a timestamp without one, fixed on both sides
E31, E32 = 1 << 31, 1 << 32
SLICE = 64 << 10  # the oracle's records come back through ctypes.string_at, whose size is a C int: < 2 GiB per slice
NTHREADS = os.cpu_count() or 8
# bench.py's RFC5424 and RFC3164 workloads (SEEDS, GEN_MEAN, DEFAULT_LINES, RFC3164_YEAR)
BENCH = {"rfc5424": (R5, 5424, 169.2, 10_000_000), "rfc3164": (R3, 3164, 140.0, 10_000_000)}
LAUNCH_LINES = 512 << 10  # the default chunk_lines: the lines of one encoder launch


def _first(mask) -> int | None:
    k = np.flatnonzero(mask)
    return int(k[0]) if len(k) else None


def _digest(view) -> bytes:
    return hashlib.blake2b(view, digest_size=16).digest()


class OracleRecords:
    """The oracle's GELF records of a batch, computed SLICE lines at a time: every record length, and one digest per
    slice of the records' bytes."""

    def __init__(self, oracle, fmt, data, offs, extra=None, cfg=None):
        self.oracle, self.fmt, self.data, self.offs, self.extra, self.cfg = oracle, fmt, data, offs, extra or {}, cfg
        self.n = len(offs) - 1
        self.cuts = list(range(0, self.n, SLICE)) + [self.n]
        self.lens = np.empty(self.n, np.int64)
        self.digests = []
        for a, b in zip(self.cuts[:-1], self.cuts[1:]):
            buf, o = self.records(a, b)
            self.lens[a:b] = np.diff(o)
            self.digests.append(_digest(buf))
        self.starts = np.zeros(self.n + 1, np.int64)
        np.cumsum(self.lens, out=self.starts[1:])
        self.total = int(self.starts[-1])

    def records(self, a, b):
        """the oracle's records of lines [a, b): (bytes, offsets rebased to the slice)"""
        return self.oracle.decode_encode_gelf(self.fmt, self.data, self.offs[a:b + 1], self.extra, cfg=self.cfg,
                                              nthreads=NTHREADS)

    def _line(self, i):
        return bytes(self.data[self.offs[i]:self.offs[i + 1]][:200])

    def _diff(self, buf, offs, i, what):
        want, wo = self.records(i, i + 1)
        got = bytes(buf[offs[i]:offs[i + 1]][:300]) if offs[i + 1] <= len(buf) else b"<past the end of the output>"
        return f"{what}: line {i}: {self._line(i)!r}\n   gpu: {got!r}\n   ref: {want[:300]!r}"

    def check(self, buf, offs, status, what):
        n = self.n
        assert len(offs) == n + 1 and len(status) == n and int(offs[0]) == 0, what
        d = np.diff(offs)
        i = _first(d < 0)
        assert i is None, f"{what}: record offsets go down at line {i}: {int(offs[i])} -> {int(offs[i + 1])}"
        assert int(offs[-1]) == self.total, f"{what}: the records end at {int(offs[-1])}, the oracle's at {self.total}"
        assert len(buf) == self.total, what
        i = _first(d != self.lens)
        assert i is None, self._diff(buf, offs, i, f"{what}: record of {int(d[i])} bytes, the oracle's has {int(self.lens[i])}")
        i = _first((status != 0) != (self.lens == 0))
        assert i is None, f"{what}: line {i}: status {int(status[i])}, oracle record of {int(self.lens[i])} bytes: {self._line(i)!r}"
        spans = [(int(offs[a]), int(offs[b])) for a, b in zip(self.cuts[:-1], self.cuts[1:])]
        with ThreadPoolExecutor(NTHREADS) as ex:
            got = list(ex.map(lambda s: _digest(buf[s[0]:s[1]]), spans))
        for k, (g, w) in enumerate(zip(got, self.digests)):
            if g == w:
                continue
            a, b = self.cuts[k], self.cuts[k + 1]
            want, wo = self.records(a, b)
            for i in range(a, b):
                if bytes(buf[offs[i]:offs[i + 1]]) != want[wo[i - a]:wo[i - a + 1]]:
                    raise AssertionError(self._diff(buf, offs, i, what))
            raise AssertionError(f"{what}: the bytes of lines [{a}, {b}) differ from the oracle's")


def _pack(lines, n, total):
    """lines (an iterable of n bytes objects, `total` bytes in all) -> (bytes uint8[total], offsets int32[n+1])"""
    data = np.empty(total, np.uint8)
    offs = np.empty(n + 1, np.int32)
    mv = memoryview(data)
    o = 0
    offs[0] = 0
    for i, line in enumerate(lines):
        mv[o:o + len(line)] = line
        o += len(line)
        offs[i + 1] = o
    assert o == total and i == n - 1
    return data, offs


def _rec_len(oracle, fmt, line, cfg=None):
    d, o = oracle.pack([line])
    buf, oo = oracle.decode_encode_gelf(fmt, d, o, cfg=cfg, nthreads=1)
    assert len(buf) > 0, line[:100]
    return len(buf)


def _tune(n, r0, targets):
    """Extra bytes per line (0 or 1) such that, with records of r0 + extra[i] bytes, one record starts exactly at each
    offset of `targets` (ascending).  Returns (extra, the line whose record starts at each target)."""
    extra = np.zeros(n, np.int64)
    j0, s0, lines = 0, 0, []
    for s in targets:
        j = j0 + (s - s0) // r0
        need = (s - s0) - (j - j0) * r0  # < r0, spread over the j - j0 lines before line j
        assert j < n and need <= j - j0
        extra[j0:j0 + need] = 1
        lines.append(j)
        j0, s0 = j, s
    return extra, lines


# Escape-heavy message: 18 of every 20 bytes are '"' or '\', every one of them escaped in short_message and full_message
MSG = (b'"\\' * 9 + b"ab") * 115
TS5 = V.TS.encode()


def _line5(i, extra):
    # the msgid appears only in full_message, unescaped: one more msgid byte moves every later record by one byte
    return b"<13>1 %s host%07d a p %s - %s" % (TS5, i, b"m" * (8 + extra), MSG)


def _line3(i, extra):
    # the blanks between the time and the host appear only in full_message: one more moves every later record by one byte
    return b"<13>Aug  6 11:15:24%s host%07d app: %s" % (b" " * (1 + extra), i, MSG)


EDGES = {"on": (E31, E32), "straddle": (E31 - 1, E32 - 1)}


def _edge_batch(oracle, fmt, line_of, edges, cfg=None):
    """One launch of LAUNCH_LINES escape-heavy lines whose records start exactly at `edges` (with "on", the record
    before the second one ends exactly at 2^32; with "straddle", the records starting one byte below 2^31 and 2^32 cross
    them).  Returns (data, offs, the lines of the edges)."""
    n = LAUNCH_LINES
    r0 = _rec_len(oracle, fmt, line_of(0, 0), cfg)
    # the tuning premise, checked on the oracle: every record of a line without extra has r0 bytes, one extra adds one
    assert _rec_len(oracle, fmt, line_of(n - 1, 0), cfg) == r0
    assert _rec_len(oracle, fmt, line_of(n - 1, 1), cfg) == r0 + 1
    extra, at = _tune(n, r0, edges)
    base = len(line_of(0, 0))
    data, offs = _pack((line_of(i, int(extra[i])) for i in range(n)), n, n * base + int(extra.sum()))
    return data, offs, at


def _small_batch(fmt):
    if fmt == R5:
        lines = [V.G1_LINE.encode(), V.G2_LINE.encode()] + [l.encode() for l, _ in V.RFC5424_CASES]
    else:
        lines = [l.encode() for _, _, l, _ in V.RFC3164_GOLDEN] + [l.encode() for l, _ in V.RFC3164_CASES]
    return lines


def _after_big_call(dec, oracle, native, fmt, cfg):
    """The context that just made a call past 2^32 (output buffer regrown, a large enc_base left behind) encodes a small
    batch exactly as the oracle and a fresh context do."""
    data, offs = oracle.pack(_small_batch(fmt))
    dec.set_gelf_extra({})
    buf, o, st, _ = dec.decode_encode_gelf(data, offs)
    want, wo = oracle.decode_encode_gelf(fmt, data, offs, cfg=cfg, nthreads=NTHREADS)
    assert buf == want and np.array_equal(o, wo)
    fresh = native.BatchDecoder(fmt, max_batch_bytes=1 << 20, max_batch_lines=1 << 12, rfc3164_year=YEAR if fmt == R3 else 0)
    try:
        fbuf, fo, fst, _ = fresh.decode_encode_gelf(data, offs)
    finally:
        fresh.close()
    assert buf == fbuf and np.array_equal(o, fo) and np.array_equal(st, fst)


_EDGE_BYTES = 1_300_000_000  # max_batch_bytes of the edge contexts: the batches of _edge_batch are about 1.24 GB


@pytest.fixture(scope="module")
def cfg3(oracle):
    return oracle.Rfc3164Config(YEAR)


@pytest.fixture
def new_ctx(native):
    """contexts closed at teardown, after a failure has been reported: the views a check takes of their pinned buffers
    are still valid when the report shows them"""
    made = []

    def make(fmt, **kw):
        made.append(native.BatchDecoder(fmt, rfc3164_year=YEAR if fmt == R3 else 0, **kw))
        return made[-1]

    yield make
    for d in made:
        d.close()


@pytest.fixture(scope="module")
def edge_ctx(native):
    """one context per source for the edge batches, default chunk_lines and default output buffer"""
    ctx = {}

    def get(fmt):
        if fmt not in ctx:
            ctx[fmt] = native.BatchDecoder(fmt, max_batch_bytes=_EDGE_BYTES, max_batch_lines=LAUNCH_LINES + 64,
                                           rfc3164_year=YEAR if fmt == R3 else 0)
        return ctx[fmt]

    yield get
    for d in ctx.values():
        d.close()


def _check_edges(dec, oracle, native, fmt, line_of, edges, cfg):
    data, offs, at = _edge_batch(oracle, fmt, line_of, EDGES[edges], cfg)
    assert int(offs[-1]) <= _EDGE_BYTES
    ora = OracleRecords(oracle, fmt, data, offs, cfg=cfg)
    # the batch reaches the edges: the oracle's records start where the layout put them, and the launch's output ends at
    # least 256 MiB past 2^32, above the default output buffer (2 x max_batch_bytes + 200 B per line), which must regrow
    assert [int(ora.starts[j]) for j in at] == list(EDGES[edges])
    assert ora.total >= E32 + (256 << 20)
    assert ora.total > 2 * _EDGE_BYTES + 200 * (LAUNCH_LINES + 64)
    assert (ora.lens > 0).all()
    dec.set_gelf_extra({})
    buf, o, st, _ = dec.decode_encode_gelf(data, offs, copy=False)
    ora.check(buf, o, st, f"one launch, records {edges} 2^31 and 2^32")
    del buf, o, st
    _after_big_call(dec, oracle, native, fmt, cfg)


@pytest.mark.parametrize("edges", sorted(EDGES))
def test_rfc5424_one_launch_past_4gib(edge_ctx, oracle, native, edges):
    _check_edges(edge_ctx(R5), oracle, native, R5, _line5, edges, None)


def test_rfc3164_one_launch_past_4gib(edge_ctx, oracle, native, cfg3):
    _check_edges(edge_ctx(R3), oracle, native, R3, _line3, "straddle", cfg3)


def test_generated_one_launch_past_4gib(oracle, native, new_ctx):
    """2.05 M generated RFC5424 lines of about 1 KB in one launch (SD pairs, arena values, wide rows, rejected lines),
    with and without output.gelf_extra"""
    n = 2_050_000
    data, offs = native.generate(native.FMT_RFC5424, 1150, n, mean_len=1150.0, bad_frac=0.005, nthreads=NTHREADS)
    dec = new_ctx(R5, max_batch_bytes=int(offs[-1]) + (1 << 20), max_batch_lines=n + 64, chunk_lines=n + 64)
    for extra in ({"env": "prod"}, {}):
        ora = OracleRecords(oracle, R5, data, offs, extra)
        assert ora.total > E32 and (ora.lens == 0).any()
        dec.set_gelf_extra(extra)
        buf, o, st, _ = dec.decode_encode_gelf(data, offs, copy=False)
        ora.check(buf, o, st, f"one launch of generated lines, gelf_extra {extra}")


@pytest.mark.parametrize("workload", sorted(BENCH))
def test_bench_workload(oracle, native, new_ctx, cfg3, workload):
    """bench.py's workload, framed (20 launches of the default chunk_lines) and raw (64 MiB stream chunks): the output
    passes 2^32 (RFC5424) or 2^31 (RFC3164) bytes, summed from one launch to the next"""
    fmt, seed, mean, n = BENCH[workload]
    stream, soffs = native.generate(fmt, seed, n, mean_len=mean, bad_frac=0.005, nthreads=NTHREADS, terminated=True)
    keep = stream != ord("\n")  # the generator puts no '\n' inside a line
    lines = stream[keep]
    del keep
    loffs = (soffs - np.arange(n + 1, dtype=np.int64)).astype(np.int32)
    cfg = cfg3 if fmt == R3 else None
    ora = OracleRecords(oracle, fmt, lines, loffs, cfg=cfg)
    assert ora.total > (E32 if fmt == R5 else E31)
    dec = new_ctx(fmt, max_batch_bytes=len(stream) + (1 << 20), max_batch_lines=n + 64)
    assert (n + LAUNCH_LINES - 1) // LAUNCH_LINES == 20
    buf, o, st, _ = dec.decode_encode_gelf(lines, loffs, copy=False)
    ora.check(buf, o, st, f"{workload} framed")
    buf, o, st, lo, _ = dec.split_decode_encode_gelf(stream, copy=False)
    assert np.array_equal(lo, soffs)
    ora.check(buf, o, st, f"{workload} raw stream")
