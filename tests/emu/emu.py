"""Loader of tests/emu/libfg_emu.so — the CPU emulation of the RFC5424 and LTSV device logic (TEST INFRASTRUCTURE).

The library is the product's walker sources (flowgger_b200/csrc/fg_r5fast.cuh, fg_rfc5424.cuh, fg_ltsvfast.cuh, fg_ltsv.cuh)
compiled with g++ plus drivers that replay the CTA rounds of parse5424_kernel / parse_ltsv_kernel / parse_gelf_kernel one
lane at a time.
Only tests import this module.
"""
from __future__ import annotations

import ctypes as C
import subprocess
from pathlib import Path

import numpy as np

HERE = Path(__file__).resolve().parent
REPO = HERE.parent.parent
_lib = None


def build(force: bool = False) -> Path:
    so = HERE / "libfg_emu.so"
    csrc = REPO / "flowgger_b200" / "csrc"
    srcs = [HERE / "emu_r5.cpp", HERE / "emu_ltsv.cpp", HERE / "emu_gelf.cpp", HERE / "emu_r3164.cpp", HERE / "cuda_shim.h",
            REPO / "include" / "flowgger_cuda.h", csrc / "fg_tz.cu"] + sorted(csrc.glob("*.cuh")) + sorted(csrc.glob("*.h"))
    if force or not so.exists() or any(s.stat().st_mtime > so.stat().st_mtime for s in srcs):
        subprocess.run(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-Wno-unknown-pragmas", "-o", str(so),
                        str(HERE / "emu_r5.cpp"), str(HERE / "emu_ltsv.cpp"), str(HERE / "emu_gelf.cpp"), str(HERE / "emu_r3164.cpp"),
                        # fg_tz.cu is host-only C++ (the zone-table reader / packer): the same source the product builds with nvcc
                        "-x", "c++", "-DFG_HOST_EMU=1", str(csrc / "fg_tz.cu"), "-I", str(REPO / "include")], check=True)
    return so


_lib_warp = None


def build_warp(force: bool = False) -> Path:
    """emu_r3164.cpp once more with FG_HOST_EMU_WARP: 32 host threads per warp, fg_any = a rendezvous of the lanes"""
    so = HERE / "libfg_emu_warp.so"
    csrc = REPO / "flowgger_b200" / "csrc"
    srcs = [HERE / "emu_r3164.cpp", HERE / "cuda_shim.h", REPO / "include" / "flowgger_cuda.h", csrc / "fg_tz.cu"] + \
        sorted(csrc.glob("*.cuh")) + sorted(csrc.glob("*.h"))
    if force or not so.exists() or any(s.stat().st_mtime > so.stat().st_mtime for s in srcs):
        subprocess.run(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-pthread", "-Wno-unknown-pragmas", "-DFG_HOST_EMU_WARP=1",
                        "-o", str(so), str(HERE / "emu_r3164.cpp"), "-x", "c++", "-DFG_HOST_EMU=1", str(csrc / "fg_tz.cu"),
                        "-I", str(REPO / "include")], check=True)
    return so


def lib_warp() -> C.CDLL:
    global _lib_warp
    if _lib_warp is None:
        _lib_warp = C.CDLL(str(build_warp()))
        _lib_warp.emu_r3164_decode.argtypes = [C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_void_p, C.c_int32, C.c_char_p,
                                               C.c_uint32, C.c_int32, C.c_void_p, C.c_void_p]
    return _lib_warp


def lib() -> C.CDLL:
    global _lib
    if _lib is None:
        _lib = C.CDLL(str(build()))
        _lib.emu5424_classify16.restype = C.c_uint32
        _lib.emu5424_classify16.argtypes = [C.c_void_p]
        _lib.emu_ltsv_classify16.restype = C.c_uint32
        _lib.emu_ltsv_classify16.argtypes = [C.c_void_p]
        _lib.emu_gelf_bits16.argtypes = [C.c_void_p, C.c_void_p]
        _lib.emu_r3164_decode.argtypes = [C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_void_p, C.c_int32, C.c_char_p,
                                          C.c_uint32, C.c_int32, C.c_void_p, C.c_void_p]
    return _lib


def classify16(block: bytes) -> int:
    assert len(block) == 16
    buf = C.create_string_buffer(block, 16)
    return int(lib().emu5424_classify16(buf))


def decode_dump(native, data: np.ndarray, offsets: np.ndarray, tile_bytes: int = 13312, strip_eol: int = 0,
                invalid: np.ndarray | None = None):
    """Emulated RFC5424 decode -> (canonical dumps, dump offsets, FgBatchOut fields as a dict) through the product's
    host materialiser (fgh_dump_records)."""
    from flowgger_b200.native import FgBatchOut, dump_records
    out = FgBatchOut()
    n = len(offsets) - 1
    lib().emu5424_decode(C.c_void_p(data.ctypes.data), C.c_void_p(offsets.ctypes.data), n, tile_bytes, int(strip_eol),
                         C.c_void_p(invalid.ctypes.data) if invalid is not None else None, C.byref(out))
    try:
        buf, offs = dump_records(native.FMT_RFC5424, out, data, offsets)
        info = {"n_entries8": out.n_entries8, "n_wide": out.n_wide, "arena_bytes": out.arena_bytes, "n_entries": out.n_entries}
        # the batch line of every wide row (WideRow.line, the first int32 of each 72-byte row)
        rows = np.ctypeslib.as_array(C.cast(out.wide_rows, C.POINTER(C.c_int32)), shape=(out.n_wide * 18,)) if out.n_wide else []
        info["wide_lines"] = {int(x) for x in rows[::18]}
    finally:
        lib().emu5424_free(C.byref(out))
    return buf, offs, info


LTSV_TYPES = {"string": 0, "bool": 1, "f64": 2, "i64": 3, "u64": 4}


def ltsv_classify16(block: bytes) -> tuple[int, int]:
    """(TAB mask, ':' mask) of a 16-byte granule."""
    assert len(block) == 16
    buf = C.create_string_buffer(block, 16)
    v = int(lib().emu_ltsv_classify16(buf))
    return v & 0xFFFF, v >> 16


def ltsv_decode_dump(native, data: np.ndarray, offsets: np.ndarray, schema: dict | None = None, suffixes: dict | None = None,
                     tile_bytes: int = 28160, strip_eol: int = 0, invalid: np.ndarray | None = None):
    """Emulated LTSV decode -> (canonical dumps, dump offsets, info dict) through the product's host materialiser."""
    from flowgger_b200.native import FgBatchOut, dump_records
    out = FgBatchOut()
    n = len(offsets) - 1
    items = list((schema or {}).items())
    names = (C.c_char_p * max(len(items), 1))(*[k.encode() for k, _ in items])
    types = (C.c_int32 * max(len(items), 1))(*[LTSV_TYPES[v.lower()] for _, v in items])
    suf = [None] * 5
    for k, v in (suffixes or {}).items():
        suf[LTSV_TYPES[k.lower()]] = v.encode()
    csuf = (C.c_char_p * 5)(*suf)
    info = (C.c_int32 * 3)()
    lib().emu_ltsv_decode(C.c_void_p(data.ctypes.data), C.c_void_p(offsets.ctypes.data), n, tile_bytes, strip_eol,
                          C.c_void_p(invalid.ctypes.data) if invalid is not None else None, 1 if schema is not None else 0,
                          len(items), names, types, csuf, C.byref(out), info)
    try:
        buf, offs = dump_records(native.FMT_LTSV, out, data, offsets, ltsv_suffix=suf)
        d = {"n_entries": out.n_entries, "rounds": int(info[0]), "direct": int(info[1]), "schema_staged": bool(info[2])}
    finally:
        lib().emu_ltsv_free(C.byref(out))
    return buf, offs, d


def r3164_decode_dump(native, data: np.ndarray, offsets: np.ndarray, year: int, tile_bytes: int = 8192, strip_eol: int = 0,
                      invalid: np.ndarray | None = None, arena_cap: int = 1 << 20, tzdir: str | None = None, lockstep: bool = True,
                      warp: bool = False):
    """Emulated RFC3164 decode -> (canonical dumps, dump offsets, info dict) through the product's host materialiser.
    warp=True: the 32-threads-per-warp build (info gains the rendezvous counts)."""
    from flowgger_b200.native import FgBatchOut, dump_records
    L = lib_warp() if warp else lib()
    out = FgBatchOut()
    n = len(offsets) - 1
    info = (C.c_int32 * 5)()
    rc = L.emu_r3164_decode(C.c_void_p(data.ctypes.data), C.c_void_p(offsets.ctypes.data), n, tile_bytes, strip_eol,
                            C.c_void_p(invalid.ctypes.data) if invalid is not None else None, year,
                            tzdir.encode() if tzdir else None, arena_cap, 1 if lockstep else 0, C.byref(out), info)
    assert rc == 0, "no zone database"
    try:
        buf, offs = dump_records(3, out, data, offsets)
        d = {"from_tile": int(info[0]), "from_global": int(info[1]), "redo": int(info[2]), "arena_bytes": int(out.arena_bytes)}
        if warp:
            d["vote_mismatches"], d["votes"] = int(info[3]), int(info[4])
    finally:
        L.emu_r3164_free(C.byref(out))
    return buf, offs, d


def r3164_site_votes() -> dict[int, int]:
    """warp build: rendezvous per source line of fg_rfc3164.cuh since the last call"""
    L = lib_warp()
    lines = (C.c_int32 * 256)()
    counts = (C.c_int64 * 256)()
    k = L.emu_r3164_site_votes(lines, counts, 256)
    return {int(lines[i]): int(counts[i]) for i in range(k)}


def tz_lookup(name: str, local: int, tzdir: str | None = None):
    """The packed zone table as the kernel searches it: UTC offset of `name` at the local second, or None."""
    L = lib()
    L.emu_tz_lookup.argtypes = [C.c_char_p, C.c_char_p, C.c_int64, C.POINTER(C.c_int32)]
    off = C.c_int32()
    rc = L.emu_tz_lookup(tzdir.encode() if tzdir else None, name.encode(), local, C.byref(off))
    assert rc >= 0, "no zone database"
    return int(off.value) if rc == 1 else None


def tz_count(tzdir: str | None = None) -> int:
    L = lib()
    L.emu_tz_count.argtypes = [C.c_char_p]
    return int(L.emu_tz_count(tzdir.encode() if tzdir else None))


def gelf_bits16(block: bytes) -> tuple[int, int, int, int]:
    """(quote mask, backslash mask, comma mask, control-byte flag) of a 16-byte granule."""
    assert len(block) == 16
    buf = C.create_string_buffer(block, 16)
    out = (C.c_uint32 * 4)()
    lib().emu_gelf_bits16(buf, out)
    return int(out[0]), int(out[1]), int(out[2]), int(out[3])


def gelf_decode_dump(native, data: np.ndarray, offsets: np.ndarray, tile_bytes: int = 34304, strip_eol: int = 0,
                     invalid: np.ndarray | None = None):
    """Emulated GELF decode -> (canonical dumps, dump offsets, info dict) through the product's host materialiser."""
    from flowgger_b200.native import FgBatchOut, dump_records
    out = FgBatchOut()
    n = len(offsets) - 1
    info = (C.c_int32 * 3)()
    lib().emu_gelf_decode(C.c_void_p(data.ctypes.data), C.c_void_p(offsets.ctypes.data), n, tile_bytes, strip_eol,
                          C.c_void_p(invalid.ctypes.data) if invalid is not None else None, C.byref(out), info)
    try:
        buf, offs = dump_records(native.FMT_GELF, out, data, offsets)
        d = {"n_entries": out.n_entries, "rounds": int(info[0]), "slow": int(info[1]), "bound_violations": int(info[2])}
    finally:
        lib().emu_gelf_free(C.byref(out))
    return buf, offs, d
