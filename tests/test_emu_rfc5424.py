"""CPU check of the RFC5424 DEVICE LOGIC: the product's walker sources (stage-1 SWAR classification, stage-2 bit-walk,
row staging, unescape, wide path) compiled with g++ (tests/emu) and replayed CTA by CTA, pushed through the product's
host materialiser and compared with the oracle.  No GPU needed; the `-m gpu` tests repeat all of this on the device."""
import numpy as np
import pytest

import vectors as V
from conftest import first_diff

R5 = 0


@pytest.fixture(scope="module")
def emu():
    import sys
    from pathlib import Path
    sys.path.insert(0, str(Path(__file__).resolve().parent / "emu"))
    import emu as E
    E.build()
    return E


def check(emu, native, oracle, data, offs, **kw):
    gbuf, goffs, info = emu.decode_dump(native, data, offs, **kw)
    obuf, ooffs = oracle.decode_dump(R5, data, offs, None, nthreads=8)
    if not (gbuf == obuf and np.array_equal(goffs, ooffs)):
        diffs = first_diff(gbuf, goffs, obuf, ooffs, data, offs)
        msg = "\n".join(f"line {i}: {line!r}\n   emu: {g!r}\n   ref: {o!r}" for i, line, g, o in diffs)
        raise AssertionError(f"{len(diffs)}+ lines differ from the oracle:\n{msg}")
    return info


def test_stage1_classification_per_byte(emu):
    """r5_classify16 flags exactly: b <= 0x22, (b & 0x1E) == 0x1C, b >= 0x7F — for every byte value in every position."""
    want = lambda b: b <= 0x22 or (b & 0x1E) == 0x1C or b >= 0x7F
    rng = np.random.default_rng(5)
    for b in range(256):
        for pos in range(16):
            blk = bytearray(rng.integers(0x30, 0x3A, 16, dtype=np.uint8).tobytes())  # digits: never flagged
            blk[pos] = b
            assert emu.classify16(bytes(blk)) == ((1 << pos) if want(b) else 0), (b, pos)
    for _ in range(2000):
        blk = rng.integers(0, 256, 16, dtype=np.uint8).tobytes()
        assert emu.classify16(blk) == sum(1 << k for k in range(16) if want(blk[k]))
    # every byte the grammar treats specially is flagged; everything unflagged is a legal SD-NAME character
    for b in b' "=]\\':
        assert want(b)
    for b in range(256):
        if not want(b):
            assert 33 <= b <= 126 and b not in b'"=]'


def test_goldens_and_appendix(emu, native, oracle):
    lines = [V.G1_LINE.encode(), V.G2_LINE.encode()] + [l.encode() for l, _ in V.RFC5424_CASES]
    data, offs = oracle.pack(lines)
    info = check(emu, native, oracle, data, offs)
    assert info["arena_bytes"] > 0  # G1/G2 hold escaped values: unescaped by the device logic


def test_generated(emu, native, oracle):
    data, offs = native.generate(native.FMT_RFC5424, 5424, 120_000, bad_frac=0.01)
    info = check(emu, native, oracle, data, offs)
    assert info["n_entries8"] > 100_000 and info["arena_bytes"] > 0
    data, offs = native.generate(native.FMT_RFC5424, 99, 40_000, bad_frac=1.0)
    check(emu, native, oracle, data, offs)


def test_small_tile_rounds_and_wide(emu, native, oracle):
    """a tile smaller than a CTA's span forces several rounds; lines longer than the tile, >= 64 KiB, or with more rows
    than fit behind the cursor go through the wide path"""
    data, offs = native.generate(native.FMT_RFC5424, 11, 5000, bad_frac=0.02)
    info = check(emu, native, oracle, data, offs, tile_bytes=256)
    assert info["n_wide"] > 0  # lines longer than the 256-byte tile
    dense = b"<13>1 " + V.TS.encode() + b" h a p m [i " + b" ".join(b'a="' + bytes([97 + k % 26]) + b'"' for k in range(40)) + b"] m"
    esc = b"<13>1 " + V.TS.encode() + b' h a p m [i a="\\"" b="\\\\" c="\\]" d="\\x" e="x\\"] m'
    lines = [V.G1_LINE.encode(), dense, esc, b"<13>1 " + V.TS.encode() + b" h a p m - " + b"x" * 70_000,
             b"<13>1 " + V.TS.encode() + b" " + b"h" * 66_000 + b' a p m [id k="v\\"w"] z', V.G2_LINE.encode()] * 3
    data, offs = oracle.pack(lines)
    info = check(emu, native, oracle, data, offs, tile_bytes=100 * 1024)
    assert info["n_wide"] >= 9 and info["n_entries"] > 0


def test_mutation_fuzz(emu, native, oracle):
    rng = np.random.default_rng(4242)
    data, offs = native.generate(native.FMT_RFC5424, 7, 30_000, bad_frac=0.0)
    alphabet = b' []"\\=<>-1:TZ+.\t!|}'
    out = []
    for i in range(len(offs) - 1):
        ln = bytearray(data[offs[i]:offs[i + 1]])
        if any(b >= 0x80 for b in ln):
            out.append(bytes(ln))
            continue
        for _ in range(int(rng.integers(1, 4))):
            k = int(rng.integers(0, len(ln)))
            op = int(rng.integers(0, 3))
            c = alphabet[int(rng.integers(0, len(alphabet)))]
            if op == 0:
                ln[k] = c
            elif op == 1:
                ln.insert(k, c)
            elif len(ln) > 1:
                del ln[k]
        out.append(bytes(ln))
    d2, o2 = oracle.pack(out)
    check(emu, native, oracle, d2, o2)


def test_split_mode_terminators(emu, native, oracle):
    lines = [V.G1_LINE.encode(), V.G2_LINE.encode(), b"", b"abc"]
    d0, o0 = oracle.pack(lines)
    obuf, ooffs = oracle.decode_dump(R5, d0, o0, None)
    want = [obuf[ooffs[i]:ooffs[i + 1]] for i in range(len(lines))]
    for mode, term in ((True, [b"\n", b"\r\n"]), (2, [b"\0", b"\0"])):
        raw = [l + term[k % 2] for k, l in enumerate(lines)]
        data, offs = oracle.pack(raw)
        gbuf, goffs, _ = emu.decode_dump(native, data, offs, strip_eol=mode)
        # spans differ by construction (terminators inside the stream); the decoded Records must not
        assert [gbuf[goffs[i]:goffs[i + 1]] for i in range(len(lines))] == want
        inv = np.array([0, 1, 0, 0], dtype=np.uint8)
        gbuf, goffs, _ = emu.decode_dump(native, data, offs, strip_eol=mode, invalid=inv)
        assert gbuf[goffs[1]:goffs[2]] == b"E:Invalid UTF-8 input;out=0" and gbuf[goffs[0]:goffs[1]] == want[0]
