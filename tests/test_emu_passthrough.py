"""CPU checks of the passthrough encoder's warp copy (flowgger_b200/csrc/fg_warp_copy.cuh), compiled with g++
(tests/emu/emu_passthrough.cpp): every source and destination misalignment 0-15 and every length 0-600, lengths past
64 KiB, and header + body records, each against memcpy, with guard bytes on both sides of the destination untouched.
No GPU needed."""
import ctypes as C
import subprocess
from pathlib import Path

import numpy as np
import pytest

HERE = Path(__file__).resolve().parent
GUARD = 64


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    so = tmp_path_factory.mktemp("emu_passthrough") / "libfg_emu_passthrough.so"
    subprocess.run(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-Wall", "-Wno-unknown-pragmas", "-o", str(so),
                    str(HERE / "emu" / "emu_passthrough.cpp")], check=True)
    L = C.CDLL(str(so))
    L.emu_warp_copy.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64]
    L.emu_copy_record.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p, C.c_uint64]
    return L


def _aligned(n: int, mis: int, fill: int) -> tuple[np.ndarray, int]:
    """a buffer of n + 2 GUARD bytes whose byte GUARD sits `mis` bytes past a 16-byte boundary: (buffer, that index)"""
    raw = np.full(n + 2 * GUARD + 32, fill, np.uint8)
    at = (-raw.ctypes.data) % 16 + 16 + mis
    return raw, at


def test_every_misalignment_and_length(emu):
    rng = np.random.default_rng(5)
    payload = rng.integers(0, 256, 600 + 32, dtype=np.uint8)
    src_raw, _ = _aligned(700, 0, 0)
    dst_raw, _ = _aligned(700, 0, 0xA5)
    sbase = (-src_raw.ctypes.data) % 16 + 16
    dbase = (-dst_raw.ctypes.data) % 16 + 16
    for sm in range(16):
        s = sbase + sm
        src_raw[:] = 0x5A
        src_raw[s:s + 600] = payload[:600]
        for dm in range(16):
            d = dbase + dm
            for n in range(601):
                dst_raw[:] = 0xA5
                emu.emu_warp_copy(dst_raw.ctypes.data + d, src_raw.ctypes.data + s, n)
                ok = (np.array_equal(dst_raw[d:d + n], src_raw[s:s + n]) and not (dst_raw[:d] != 0xA5).any()
                      and not (dst_raw[d + n:] != 0xA5).any())
                assert ok, (sm, dm, n)


@pytest.mark.parametrize("n", [65535, 65536, 65537, 100_003, 1 << 20])
def test_long_spans(emu, n):
    rng = np.random.default_rng(n)
    payload = rng.integers(0, 256, n, dtype=np.uint8)
    for sm, dm in ((0, 0), (3, 0), (0, 7), (5, 11), (15, 1), (4, 8)):
        src, s = _aligned(n, sm, 0x5A)
        src[s:s + n] = payload
        dst, d = _aligned(n, dm, 0xA5)
        emu.emu_warp_copy(dst.ctypes.data + d, src.ctypes.data + s, n)
        assert np.array_equal(dst[d:d + n], payload)
        assert not (dst[:d] != 0xA5).any() and not (dst[d + n:] != 0xA5).any()


@pytest.mark.parametrize("hn,bn", [(0, 0), (0, 37), (1, 0), (13, 600), (17, 65537), (70_001, 3), (64, 100_000), (100_000, 100_000)])
def test_header_plus_body(emu, hn, bn):
    """a record as the write pass stores it: header, then body at every alignment the header leaves"""
    rng = np.random.default_rng(hn * 7 + bn)
    hdr = rng.integers(0, 256, hn, dtype=np.uint8)
    body = rng.integers(0, 256, bn, dtype=np.uint8)
    for hm, bm, dm in ((0, 0, 0), (1, 2, 3), (9, 0, 15), (0, 13, 6)):
        hb, h = _aligned(hn, hm, 0)
        hb[h:h + hn] = hdr
        bb, b = _aligned(bn, bm, 0)
        bb[b:b + bn] = body
        dst, d = _aligned(hn + bn, dm, 0xA5)
        emu.emu_copy_record(dst.ctypes.data + d, hb.ctypes.data + h, hn, bb.ctypes.data + b, bn)
        assert dst[d:d + hn + bn].tobytes() == hdr.tobytes() + body.tobytes()
        assert not (dst[:d] != 0xA5).any() and not (dst[d + hn + bn:] != 0xA5).any()
