"""CPU checks of output.framing on the fused GELF encoder: the syslen prefix writer and the framed / unframed record
lengths of fg_out_frame.cuh, compiled with g++ (tests/emu/emu_frame.cpp), against Python's decimal text at every
power-of-ten edge of a 64-bit length and on random lengths; and the merger restatement (tests/merger_oracle.py) against
the reference's mergers.  No GPU needed."""
import ctypes as C
import subprocess
from pathlib import Path

import numpy as np
import pytest

import merger_oracle as M

HERE = Path(__file__).resolve().parent


@pytest.fixture(scope="module")
def frame(tmp_path_factory):
    so = tmp_path_factory.mktemp("emu_frame") / "libfg_emu_frame.so"
    subprocess.run(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-Wno-unknown-pragmas", "-o", str(so),
                    str(HERE / "emu" / "emu_frame.cpp")], check=True)
    L = C.CDLL(str(so))
    L.emu_syslen_prefix.argtypes = [C.c_uint64, C.c_void_p]
    L.emu_syslen_prefix.restype = C.c_int
    L.emu_framed_len.argtypes = [C.c_uint64, C.c_int]
    L.emu_framed_len.restype = C.c_uint64
    L.emu_unframed_len.argtypes = [C.c_uint64, C.c_int]
    L.emu_unframed_len.restype = C.c_uint64
    L.emu_write_framed.argtypes = [C.c_char_p, C.c_uint64, C.c_int, C.c_void_p]
    return L


def _lengths():
    """L with L + 1 at 10^k - 2 ... 10^k + 1 for every k up to 2^63, 2^32 and 2^63 neighbours, and random 64-bit values"""
    out = set()
    for k in range(1, 20):
        for d in (-2, -1, 0, 1):
            m = 10 ** k + d
            if 1 <= m <= 2 ** 63:
                out.add(m - 1)
    out.update({0, 1, 2 ** 32 - 2, 2 ** 32 - 1, 2 ** 32, 2 ** 63 - 2, 2 ** 63 - 1})
    rng = np.random.default_rng(64)
    out.update(int(v) for v in rng.integers(0, 2 ** 63 - 1, size=5000, dtype=np.int64))
    out.update(int(v) >> int(s) for v, s in zip(rng.integers(0, 2 ** 63 - 1, size=5000, dtype=np.int64), rng.integers(0, 63, size=5000)))
    return sorted(out)


def test_syslen_prefix_is_the_decimal_of_len_plus_one(frame):
    buf = C.create_string_buffer(32)
    for L in _lengths():
        n = frame.emu_syslen_prefix(L, buf)
        assert buf.raw[:n] == f"{L + 1} ".encode(), L


def test_framed_lengths_invert(frame):
    for L in _lengths():
        for framing in (M.NONE, M.LINE, M.NUL, M.SYSLEN):
            want = len(M.MERGERS[framing](b"")) + L if framing != M.SYSLEN else len(f"{L + 1} ") + L + 1
            f = frame.emu_framed_len(L, framing)
            assert f == want, (L, framing)
            assert frame.emu_unframed_len(f, framing) == L, (L, framing)


def test_mergers_match_the_reference():
    # line_merger.rs:14, nul_merger.rs:14, syslen_merger.rs:15-28 (format!("{} ", len + 1), record, 0x0a)
    assert M.line_merger(b'{"a":1}') == b'{"a":1}\n'
    assert M.nul_merger(b'{"a":1}') == b'{"a":1}\0'
    assert M.syslen_merger(b"") == b"1 \n"
    assert M.syslen_merger(b"x" * 8) == b"9 " + b"x" * 8 + b"\n"
    assert M.syslen_merger(b"x" * 9) == b"10 " + b"x" * 9 + b"\n"
    assert M.syslen_merger(b"x" * 99) == b"100 " + b"x" * 99 + b"\n"
    assert M.MERGERS[M.NONE](b"abc") == b"abc"
    recs, ok = [b"a", b"", b"bc"], [True, False, True]
    assert M.output_stream(recs, ok, M.NONE) == b"abc"
    assert M.output_stream(recs, ok, M.LINE) == b"a\nbc\n"
    assert M.output_stream(recs, ok, M.NUL) == b"a\0bc\0"
    assert M.output_stream(recs, ok, M.SYSLEN) == b"2 a\n3 bc\n"


def test_write_pass_frames_like_the_mergers(frame):
    """frame_record (the frame the write pass stores around a record's place) + the record's bytes = the merger's
    output, for record lengths around every syslen digit edge that a test can hold in memory"""
    rng = np.random.default_rng(7)
    for L in sorted({0, 1, 2, 7, 8, 9, 10, 11, 97, 98, 99, 100, 998, 999, 1000, 9998, 9999, 10000, 99999, 100000,
                     *rng.integers(0, 300000, size=40).tolist()}):
        rec = bytes(rng.integers(0, 256, size=L, dtype=np.uint8))
        for framing in (M.NONE, M.LINE, M.NUL, M.SYSLEN):
            want = M.MERGERS[framing](rec)
            out = C.create_string_buffer(len(want))
            frame.emu_write_framed(rec, L, framing, out)
            assert out.raw == want, (L, framing)
