"""RFC3164 on the device (SURVEY.md §8(f) N3): parse3164_kernel through the C ABI against the oracle.
(The file sorts last on purpose: the format was added last, so the older formats' GPU tests run first.)"""
import numpy as np
import pytest

import vectors as V
from conftest import assert_parity

pytestmark = pytest.mark.gpu
R3 = 3
YEAR = 2026


@pytest.fixture(scope="module")
def dec(native):
    d = native.BatchDecoder(native.FMT_RFC3164, max_batch_bytes=96 << 20, max_batch_lines=1 << 20, rfc3164_year=YEAR)
    yield d
    d.close()


def test_goldens_and_derived_cases(dec, native, oracle):
    lines = [l.encode() for _, _, l, _ in V.RFC3164_GOLDEN] + [l.encode() for l, _ in V.RFC3164_CASES]
    data, offs = oracle.pack(lines)
    for year in (2026, 2024):
        dec.set_rfc3164_year(year)
        res = assert_parity(dec, oracle, R3, data, offs, oracle.Rfc3164Config(year))
    dec.set_rfc3164_year(YEAR)
    res = dec.decode(data, offs)
    n_gold = len(V.RFC3164_GOLDEN)
    for k, (line, err) in enumerate(V.RFC3164_CASES):
        st = int(res.status[n_gold + k])
        assert (native.error_string(R3, st) if st else None) == err, (line, st)
    assert dec.kernel_launches() >= 1


def test_generated_and_resident(dec, native, oracle):
    cfg = oracle.Rfc3164Config(YEAR)
    data, offs = native.generate(native.FMT_RFC3164, 3164, 600_000, bad_frac=0.02)
    res = assert_parity(dec, oracle, R3, data, offs, cfg)
    assert len(res.arena) > 100_000                  # re-joined messages came back from the device arena
    assert_parity(dec, oracle, R3, data, offs, cfg, resident=True)
    data, offs = native.generate(native.FMT_RFC3164, 31, 50_000, bad_frac=1.0)
    assert_parity(dec, oracle, R3, data, offs, cfg)
    data, offs = native.generate(native.FMT_RFC3164, 64, 50_000, mean_len=900.0)
    assert_parity(dec, oracle, R3, data, offs, cfg)


def test_arena_regrow_long_lines_and_zones(native, oracle):
    cfg = oracle.Rfc3164Config(YEAR)
    d = native.BatchDecoder(native.FMT_RFC3164, max_batch_bytes=1 << 20, max_batch_lines=1 << 12, rfc3164_year=YEAR)
    try:
        # max_batch_bytes / 32 = 32 KiB of arena at first: 1.2 MB of irregularly spaced messages force regrow + redo
        long_line = b"<13>Aug  6 11:15:24 host tag: " + b"x y  " * 20_000
        lines = [long_line, b"<13>Aug  6 11:15:24 host tag: short", long_line[:70_000]] + [b"Aug 6 11:15:24 h a  b\tc"] * 3000
        data, offs = oracle.pack(lines)
        assert_parity(d, oracle, R3, data, offs, cfg)
        import tzread
        names = sorted(tzread.load_zones())
        lines = []
        for k, nm in enumerate(names):
            lines.append(f"<{k % 192}>{1990 + k % 60} Mar {1 + k % 28} 0{k % 10}:30:00 {nm} host tag: m {k}".encode())
            lines.append(f"Oct 31 01:30:00 {nm[:-1]} host m".encode())
            lines.append(f"h{k}: 2031 Nov 2 01:30:00 {nm}: m".encode())
        data, offs = oracle.pack(lines)
        assert_parity(d, oracle, R3, data, offs, cfg)
        # a caller-supplied zone table replaces the system database (fg_set_tz_table)
        mine = {"Mars/Phobos": ([0, 1_000_000_000], [3600, 7200, -1800]), "UTC": ([], [0])}
        d.set_tz_table(mine)
        data, offs = oracle.pack([b"2020 Aug 6 11:15:24 Mars/Phobos h m", b"1980 Aug 6 11:15:24 Mars/Phobos h m",
                                  b"2020 Aug 6 11:15:24 Europe/Paris h m", b"Aug 6 11:15:24 UTC h m"])
        assert_parity(d, oracle, R3, data, offs, oracle.Rfc3164Config(YEAR, mine))
    finally:
        d.close()


def test_split_decode_and_decoder_trait(dec, native, oracle):
    cfg = oracle.Rfc3164Config(YEAR)
    import pysplit
    data, _ = native.generate(native.FMT_RFC3164, 77, 100_000, bad_frac=0.02, terminated=True)
    stream = bytes(data)
    stream = stream[:5000] + b"\xfe" + stream[5000:]        # one record that is not UTF-8: reported, not decoded
    arr = np.frombuffer(stream, dtype=np.uint8).copy()
    loffs, lines, valid = pysplit.split_lines(stream)
    buf, bo, line_offs, _ = dec.split_dump(arr, 0)
    assert np.array_equal(line_offs, loffs)
    good = [l for l, v in zip(lines, valid) if v]
    d1, o1 = oracle.pack(good)
    obuf, oo = oracle.decode_dump(R3, d1, o1, cfg)
    k = 0
    for i, v in enumerate(valid):
        got = buf[bo[i]:bo[i + 1]]
        if not v:
            assert got == b"E:Invalid UTF-8 input;out=0", (i, got)
        else:
            assert got == obuf[oo[k]:oo[k + 1]], (i, lines[i], got, obuf[oo[k]:oo[k + 1]])
            k += 1
    assert sum(1 for v in valid if not v) == 1
    # Decoder::decode + clone_boxed from two threads (batches of one through the same kernel)
    # (lines that carry their year: the clones are built without one and follow the clock)
    some = [l.encode() for name, _, l, _ in V.RFC3164_GOLDEN if name in ("G18", "G19", "G23", "G24", "G25")] * 8
    got = native.clone_decode_threads(native.FMT_RFC3164, some, nthreads=2)
    dd, oo = oracle.pack(some)
    ob, oof = oracle.decode_dump(R3, dd, oo, cfg)
    assert got == [ob[oof[i]:oof[i + 1]] for i in range(len(some))]
