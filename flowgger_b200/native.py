"""ctypes binding of include/flowgger_cuda.h (+ the C++ host mirror and the synthetic generators)."""
from __future__ import annotations

import ctypes as C
import os
from pathlib import Path

import numpy as np

LIB_DIR = Path(__file__).resolve().parent / "lib"

FMT_RFC5424, FMT_LTSV, FMT_GELF, FMT_RFC3164 = 0, 1, 2, 3
FMT_NAMES = {FMT_RFC5424: "rfc5424", FMT_LTSV: "ltsv", FMT_GELF: "gelf", FMT_RFC3164: "rfc3164"}
# output.framing of the fused encoder (fg_out_framing)
OUT_NONE, OUT_LINE, OUT_NUL, OUT_SYSLEN = 0, 1, 2, 3


class NativeLibraryMissing(ImportError):
    pass


class FgSpan(C.Structure):
    _fields_ = [("off", C.c_int32), ("len", C.c_int32)]


class FgBatchOut(C.Structure):
    _fields_ = [
        ("n", C.c_int32), ("n_entries", C.c_int32),
        ("ts", C.POINTER(C.c_double)), ("meta", C.POINTER(C.c_uint32)),
        ("hostname", C.POINTER(FgSpan)), ("appname", C.POINTER(FgSpan)), ("procid", C.POINTER(FgSpan)),
        ("msgid", C.POINTER(FgSpan)), ("msg", C.POINTER(FgSpan)), ("full_msg", C.POINTER(FgSpan)),
        ("sd", C.POINTER(FgSpan)),
        ("entry_name", C.POINTER(FgSpan)), ("entry_val", C.POINTER(C.c_uint64)), ("entry_meta", C.POINTER(C.c_uint8)),
        ("line_offsets", C.POINTER(C.c_int32)),
        ("rows5424", C.c_void_p), ("entries8", C.POINTER(C.c_uint64)), ("n_entries8", C.c_int32), ("n_wide", C.c_int32),
        ("wide_rows", C.c_void_p), ("arena", C.POINTER(C.c_uint8)), ("arena_bytes", C.c_int64),
        ("kernel_ms", C.c_float), ("total_ms", C.c_float),
    ]


# include/flowgger_cuda.h: fg_row5424 (32 bytes) and fg_wide_row (72 bytes)
ROW5424 = np.dtype([("ts", "<f8"), ("meta", "<u4"), ("sd_first", "<u4"), ("sd_count", "<u2"), ("sp", "<u2", (5,)),
                    ("msg_off", "<u2"), ("msg_len", "<u2")])
WIDE_ROW = np.dtype([("line", "<i4"), ("meta", "<u4"), ("ts", "<f8"), ("hostname", "<i4", (2,)), ("appname", "<i4", (2,)),
                     ("procid", "<i4", (2,)), ("msgid", "<i4", (2,)), ("msg", "<i4", (2,)), ("full_msg", "<i4", (2,)),
                     ("sd", "<i4", (2,))])
assert ROW5424.itemsize == 32 and WIDE_ROW.itemsize == 72


class FgEncodedOut(C.Structure):
    _fields_ = [("n", C.c_int32), ("bytes", C.POINTER(C.c_uint8)), ("offsets", C.POINTER(C.c_int64)), ("status", C.POINTER(C.c_uint8)),
                ("kernel_ms", C.c_float), ("total_ms", C.c_float)]


_cuda = None
_host = None
_gen = None


def cuda_lib_path() -> Path:
    return LIB_DIR / "libflowgger_cuda.so"


def _load(name: str) -> C.CDLL:
    p = LIB_DIR / name
    if name == "libflowgger_cuda.so" and os.environ.get("FG_VARIANT_DIR"):
        # A/B harness for kernel-shape experiments: another build of the SAME library
        p = Path(os.environ["FG_VARIANT_DIR"]) / name
    if not p.exists():
        raise NativeLibraryMissing(
            f"{p} is missing: run `python -m flowgger_b200.build` (nvcc, sm_90a). "
            "flowgger_b200 has no CPU fallback.")
    return C.CDLL(str(p), mode=C.RTLD_GLOBAL)


def load_cuda() -> C.CDLL:
    global _cuda
    if _cuda is None:
        L = _load("libflowgger_cuda.so")
        L.fg_error_string.restype = C.c_char_p
        L.fg_error_string.argtypes = [C.c_int, C.c_uint32]
        L.fg_build_info.restype = C.c_char_p
        L.fg_last_error.restype = C.c_char_p
        L.fg_last_error.argtypes = [C.c_void_p]
        L.fg_kernel_launches.restype = C.c_int64
        L.fg_kernel_launches.argtypes = [C.c_void_p]
        L.fg_decode_batch.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_int32, C.POINTER(FgBatchOut)]
        L.fg_upload.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32]
        L.fg_parse_resident.argtypes = [C.c_void_p, C.c_int, C.POINTER(C.c_float)]
        L.fg_download.argtypes = [C.c_void_p, C.c_int, C.POINTER(FgBatchOut)]
        L.fg_parse_resident_n.argtypes = [C.c_void_p, C.c_int, C.c_int32, C.POINTER(C.c_float)]
        L.fg_flush_l2.argtypes = [C.c_void_p]
        L.fg_host_alloc.argtypes = [C.c_void_p, C.c_size_t, C.POINTER(C.c_void_p)]
        L.fg_host_free.argtypes = [C.c_void_p, C.c_void_p]
        L.fg_split_decode.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_int64, C.POINTER(FgBatchOut)]
        L.fg_split_decode_framed.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_int64, C.POINTER(FgBatchOut)]
        L.fg_last_split_ms.restype = C.c_float
        L.fg_last_split_ms.argtypes = [C.c_void_p]
        L.fg_error_count.restype = C.c_uint32
        L.fg_last_dominant_kernel_ms.restype = C.c_float
        L.fg_last_dominant_kernel_ms.argtypes = [C.c_void_p]
        L.fg_set_rfc3164_year.argtypes = [C.c_void_p, C.c_int32]
        L.fg_set_tz_table.argtypes = [C.c_void_p, C.c_int32, C.POINTER(C.c_char_p), C.c_void_p, C.c_void_p, C.c_void_p]
        L.fg_tz_lookup.argtypes = [C.c_char_p, C.c_char_p, C.c_int64, C.POINTER(C.c_int32)]
        L.fg_tz_count.argtypes = [C.c_char_p]
        L.fg_tz_count.restype = C.c_int32
        L.fg_set_gelf_extra.argtypes = [C.c_void_p, C.c_int32, C.POINTER(C.c_char_p), C.POINTER(C.c_char_p)]
        L.fg_decode_encode_gelf.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_int32, C.POINTER(FgEncodedOut)]
        L.fg_split_decode_encode_gelf.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_int64, C.POINTER(FgEncodedOut),
                                                  C.POINTER(C.POINTER(C.c_int32))]
        L.fg_set_ltsv_extra.argtypes = [C.c_void_p, C.c_int32, C.POINTER(C.c_char_p), C.POINTER(C.c_char_p)]
        L.fg_decode_encode_ltsv.argtypes = L.fg_decode_encode_gelf.argtypes
        L.fg_split_decode_encode_ltsv.argtypes = L.fg_split_decode_encode_gelf.argtypes
        L.fg_set_capnp_extra.argtypes = L.fg_set_ltsv_extra.argtypes
        L.fg_decode_encode_capnp.argtypes = L.fg_decode_encode_gelf.argtypes
        L.fg_split_decode_encode_capnp.argtypes = L.fg_split_decode_encode_gelf.argtypes
        L.fg_set_passthrough_prefix.argtypes = [C.c_void_p, C.c_char_p, C.c_int64]
        L.fg_decode_encode_passthrough.argtypes = L.fg_decode_encode_gelf.argtypes
        L.fg_split_decode_encode_passthrough.argtypes = L.fg_split_decode_encode_gelf.argtypes
        L.fg_encoded_ltsv_stops.argtypes = [C.c_void_p, C.POINTER(C.POINTER(C.c_int32))]
        L.fg_encoded_gelf_now.argtypes = [C.c_void_p, C.POINTER(C.c_double)]
        L.fg_set_output_framing.argtypes = [C.c_void_p, C.c_int]
        _cuda = L
    return _cuda


def load_host() -> C.CDLL:
    global _host
    if _host is None:
        load_cuda()
        L = _load("libflowgger_host.so")
        L.fgh_decoder_new.restype = C.c_void_p
        L.fgh_decoder_new.argtypes = [C.c_int, C.c_int, C.c_int64, C.c_int32, C.c_int32, C.c_int, C.c_int,
                                      C.POINTER(C.c_char_p), C.POINTER(C.c_char_p), C.c_int,
                                      C.POINTER(C.c_char_p), C.POINTER(C.c_char_p), C.c_char_p, C.c_int]
        L.fgh_decoder_free.argtypes = [C.c_void_p]
        L.fgh_decoder_ctx.restype = C.c_void_p
        L.fgh_decoder_ctx.argtypes = [C.c_void_p]
        L.fgh_free.argtypes = [C.c_void_p]
        L.fgh_dump_out.argtypes = [C.c_void_p, C.POINTER(FgBatchOut), C.c_void_p, C.c_void_p, C.c_int,
                                   C.POINTER(C.c_void_p), C.POINTER(C.c_void_p)]
        L.fgh_dump_range.argtypes = [C.c_void_p, C.POINTER(FgBatchOut), C.c_void_p, C.c_void_p, C.c_int64, C.c_int64, C.c_int,
                                     C.POINTER(C.c_void_p), C.POINTER(C.c_void_p)]
        L.fgh_dump_records.argtypes = [C.c_int, C.POINTER(FgBatchOut), C.c_void_p, C.c_void_p, C.c_void_p, C.POINTER(C.c_void_p),
                                       C.POINTER(C.c_void_p)]
        L.fgh_materialize_bench.restype = C.c_double
        L.fgh_materialize_bench.argtypes = [C.c_void_p, C.POINTER(FgBatchOut), C.c_void_p, C.c_void_p, C.c_int]
        L.fgh_is_valid_utf8.argtypes = [C.c_void_p, C.c_int64]
        L.fgh_split_dump.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_int64, C.POINTER(C.c_void_p), C.POINTER(C.c_void_p),
                                     C.POINTER(C.c_void_p), C.POINTER(C.c_int32), C.POINTER(C.c_float), C.c_char_p, C.c_int]
        L.fgh_shard_by_bytes.argtypes = [C.c_void_p, C.c_int32, C.c_int, C.c_void_p]
        L.fgh_multi_decode_dump.argtypes = [C.c_int, C.c_void_p, C.c_int, C.c_int64, C.c_int32, C.c_void_p, C.c_void_p,
                                            C.c_int32, C.POINTER(C.c_void_p), C.POINTER(C.c_void_p), C.c_char_p, C.c_int]
        L.fgh_clone_decode_threads.argtypes = [C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_int32, C.c_int,
                                               C.POINTER(C.c_void_p), C.POINTER(C.c_void_p), C.c_char_p, C.c_int]
        L.fgh_splitter_run_gelf.argtypes = [C.c_void_p, C.c_char_p, C.c_int64, C.c_int32, C.c_int64, C.c_int, C.POINTER(C.c_char_p),
                                            C.POINTER(C.c_char_p)] + [C.POINTER(C.c_void_p), C.POINTER(C.c_int64)] * 2 + [C.c_int] + [
                                            C.POINTER(C.c_void_p), C.POINTER(C.c_int64)]
        L.fgh_splitter_run_gelf_framed.argtypes = [C.c_void_p, C.c_char_p, C.c_int64, C.c_int32, C.c_int64, C.c_int, C.POINTER(C.c_char_p),
                                                   C.POINTER(C.c_char_p), C.c_int, C.c_int] + [C.POINTER(C.c_void_p), C.POINTER(C.c_int64)] * 3
        L.fgh_splitter_run_ltsv_framed.argtypes = L.fgh_splitter_run_gelf_framed.argtypes
        L.fgh_splitter_run_capnp_framed.argtypes = L.fgh_splitter_run_gelf_framed.argtypes
        L.fgh_splitter_run_passthrough_framed.argtypes = [C.c_void_p, C.c_char_p, C.c_int64, C.c_int32, C.c_int64, C.c_char_p, C.c_int64,
                                                          C.c_int, C.c_int] + [C.POINTER(C.c_void_p), C.POINTER(C.c_int64)] * 3
        L.fgh_splitter_run.argtypes = [C.c_void_p, C.c_int, C.c_char_p, C.c_int64, C.c_int32, C.c_int64] + [C.POINTER(C.c_void_p), C.POINTER(C.c_int64)] * 3
        _host = L
    return _host


def load_gen() -> C.CDLL:
    global _gen
    if _gen is None:
        L = _load("libfg_gen.so")
        L.fgen_generate.argtypes = [C.c_int, C.c_uint64, C.c_int64, C.c_int64, C.c_double, C.c_double, C.c_int,
                                    C.POINTER(C.c_void_p), C.POINTER(C.c_void_p), C.POINTER(C.c_int64)]
        L.fgen_free.argtypes = [C.c_void_p]
        L.fgen_set_terminator.argtypes = [C.c_int]
        _gen = L
    return _gen


def build_info() -> str:
    return load_cuda().fg_build_info().decode()


def error_string(fmt: int, status: int) -> str | None:
    s = load_cuda().fg_error_string(fmt, status)
    return None if s is None else s.decode()


def generate(fmt: int, seed: int, n: int, *, first_index: int = 0, mean_len: float = 0.0, bad_frac: float = 0.005,
             nthreads: int = 8, terminated: bool = False) -> tuple[np.ndarray, np.ndarray]:
    """Synthetic batch (SURVEY.md §8(d) shapes): returns (bytes uint8[total], offsets int32[n+1])."""
    L = load_gen()
    if mean_len <= 0:
        mean_len = {FMT_RFC5424: 180.0, FMT_GELF: 512.0, FMT_LTSV: 420.0, FMT_RFC3164: 140.0}[fmt]
    pb, po, tot = C.c_void_p(), C.c_void_p(), C.c_int64()
    L.fgen_set_terminator(1 if terminated else 0)  # terminated: every line ends in '\n' (raw stream for split_decode)
    rc = L.fgen_generate(fmt, seed, first_index, n, mean_len, bad_frac, nthreads, C.byref(pb), C.byref(po), C.byref(tot))
    if rc != 0:
        raise ValueError("generated batch exceeds the int32 offset range; generate fewer lines per batch")
    try:
        b = np.ctypeslib.as_array(C.cast(pb, C.POINTER(C.c_uint8)), shape=(max(tot.value, 1),))[: tot.value].copy()
        o = np.ctypeslib.as_array(C.cast(po, C.POINTER(C.c_int32)), shape=(n + 1,)).copy()
    finally:
        L.fgen_free(pb)
        L.fgen_free(po)
    return b, o


def _ptr(a: np.ndarray) -> C.c_void_p:
    return C.c_void_p(a.ctypes.data)


def _c_strings(xs: list[str]):
    return (C.c_char_p * max(len(xs), 1))(*[x.encode() for x in xs])


def _extra_arrays(extra: dict[str, str] | None):
    """output.gelf_extra as (count, keys, values) C string arrays."""
    ex = list((extra or {}).items())
    return len(ex), _c_strings([k for k, _ in ex]), _c_strings([v for _, v in ex])


def _take_dumps(pb: C.c_void_p, po: C.c_void_p, n: int) -> tuple[bytes, np.ndarray]:
    """Reads and frees the (buffer, int64 offsets[n + 1]) pair of canonical dumps an fgh_* entry returned."""
    H = load_host()
    try:
        offs = np.ctypeslib.as_array(C.cast(po, C.POINTER(C.c_int64)), shape=(n + 1,)).copy()
        buf = C.string_at(pb, int(offs[-1]))
    finally:
        H.fgh_free(pb)
        H.fgh_free(po)
    return buf, offs


def _encoded_views(out: FgEncodedOut):
    """Views of an fg_encoded_out: (JSON bytes, int64 offsets[n + 1], status uint8[n])."""
    n = out.n
    offs = np.ctypeslib.as_array(out.offsets, shape=(n + 1,))
    total = int(offs[-1]) if n else 0
    buf = np.ctypeslib.as_array(out.bytes, shape=(max(total, 1),))[:total]
    status = np.ctypeslib.as_array(out.status, shape=(max(n, 1),))[:n]
    return buf, offs, status


def _run_splitter(call) -> tuple[bytes, bytes, bytes]:
    """Runs a splitter entry with three malloc'd (pointer, length) outputs, `call(outs)` given their six by-reference
    arguments in order, and returns and frees the outputs."""
    H = load_host()
    ps = [C.c_void_p() for _ in range(3)]
    ns = [C.c_int64() for _ in range(3)]
    if call([a for p, n in zip(ps, ns) for a in (C.byref(p), C.byref(n))]) != 0:
        raise RuntimeError("splitter failed")
    out = []
    for p, n in zip(ps, ns):
        out.append(C.string_at(p, n.value))
        H.fgh_free(p)
    return tuple(out)


class BatchResult:
    """numpy views over one fg_batch_out (valid until the next decode on the same decoder)."""

    def __init__(self, out: FgBatchOut, fmt: int):
        self.raw = out
        self.fmt = fmt
        self.n = out.n
        self.n_entries = out.n_entries
        self.kernel_ms = out.kernel_ms
        self.total_ms = out.total_ms
        n, ne = out.n, out.n_entries

        def arr(p, dtype, count, cols=None):
            if not p or count == 0:
                return np.zeros((0,) if cols is None else (0, cols), dtype=dtype)
            if isinstance(p, int):
                p = C.c_void_p(p)
            a = np.ctypeslib.as_array(C.cast(p, C.POINTER(C.c_uint8)), shape=(count * np.dtype(dtype).itemsize * (cols or 1),))
            a = a.view(dtype)
            return a if cols is None else a.reshape(count, cols)

        # RFC5424: compact rows (the columns below are derived views / empty)
        self.rows5424 = arr(out.rows5424, ROW5424, n)
        self.entries8 = arr(out.entries8, np.uint64, out.n_entries8)
        self.wide_rows = arr(out.wide_rows, WIDE_ROW, out.n_wide)
        self.arena = arr(out.arena, np.uint8, out.arena_bytes)
        if fmt == FMT_RFC5424:
            self.ts = self.rows5424["ts"] if n else np.zeros(0)
            self.meta = self.rows5424["meta"] if n else np.zeros(0, np.uint32)
            for name in ("hostname", "appname", "procid", "msgid", "msg", "full_msg", "sd"):
                setattr(self, name, np.zeros((0, 2), np.int32))
            self.entry_name = arr(out.entry_name, np.int32, ne, 2)
            self.entry_val = arr(out.entry_val, np.uint64, ne)
            self.entry_meta = arr(out.entry_meta, np.uint8, ne)
            return
        self.ts = arr(out.ts, np.float64, n)
        self.meta = arr(out.meta, np.uint32, n)
        self.hostname = arr(out.hostname, np.int32, n, 2)
        self.appname = arr(out.appname, np.int32, n, 2)
        self.procid = arr(out.procid, np.int32, n, 2)
        self.msgid = arr(out.msgid, np.int32, n, 2)
        self.msg = arr(out.msg, np.int32, n, 2)
        self.full_msg = arr(out.full_msg, np.int32, n, 2)
        self.sd = arr(out.sd, np.int32, n, 2)
        self.entry_name = arr(out.entry_name, np.int32, ne, 2)
        self.entry_val = arr(out.entry_val, np.uint64, ne)
        self.entry_meta = arr(out.entry_meta, np.uint8, ne)

    @property
    def status(self) -> np.ndarray:
        return self.meta & 0xFF

    def spans5424(self, offsets: np.ndarray) -> dict[str, np.ndarray]:
        """RFC5424 compact rows -> absolute (off, len) spans like the fg_row5424_* helpers of the C header (rows that are
        errors or FG_FLAG_WIDE get off = -1)."""
        r = self.rows5424
        lo = offsets[:-1].astype(np.int64)
        flags = r["meta"] >> 24
        good = ((r["meta"] & 0xFF) == 0) & ((flags & 0x80) == 0)
        sp = r["sp"].astype(np.int64)
        out = {}
        for k, name in enumerate(("hostname", "appname", "procid", "msgid")):
            out[name] = np.stack([np.where(good, lo + sp[:, k] + 1, -1), np.where(good, sp[:, k + 1] - sp[:, k] - 1, 0)], axis=1)
        mo, ml = r["msg_off"].astype(np.int64), r["msg_len"].astype(np.int64)
        out["msg"] = np.stack([np.where(good & (ml > 0), lo + mo, -1), np.where(good, ml, 0)], axis=1)
        out["full_msg"] = np.stack([np.where(good, lo, -1), np.where(good, mo + ml, 0)], axis=1)
        out["sd"] = np.stack([r["sd_first"].astype(np.int64), np.where(good, r["sd_count"].astype(np.int64), 0)], axis=1)
        return out


class BatchDecoder:
    """One GPU decoding context of a fixed format (wraps flowgger::CudaBatchDecoder / fg_ctx)."""

    def __init__(self, fmt: int, *, device: int = 0, max_batch_bytes: int = 0, max_batch_lines: int = 0,
                 chunk_lines: int = 0, ltsv_schema: dict[str, str] | None = None,
                 ltsv_suffixes: dict[str, str] | None = None, rfc3164_year: int = 0):
        self._h = None
        self.L = load_cuda()
        self.H = load_host()
        self.fmt = fmt
        schema = list((ltsv_schema or {}).items())
        suff = list((ltsv_suffixes or {}).items())
        err = C.create_string_buffer(512)
        h = self.H.fgh_decoder_new(fmt, device, max_batch_bytes, max_batch_lines, chunk_lines,
                                   1 if ltsv_schema is not None else 0, len(schema),
                                   _c_strings([k for k, _ in schema]), _c_strings([v for _, v in schema]), len(suff),
                                   _c_strings([k for k, _ in suff]), _c_strings([v for _, v in suff]), err, 512)
        if not h:
            raise RuntimeError(err.value.decode() or "fgh_decoder_new failed")
        self._h = C.c_void_p(h)
        self.ctx = C.c_void_p(self.H.fgh_decoder_ctx(self._h))
        self._pinned: list[C.c_void_p] = []
        if rfc3164_year:
            self.set_rfc3164_year(rfc3164_year)

    def set_rfc3164_year(self, year: int) -> None:
        """The year a timestamp without one belongs to (`OffsetDateTime::now_utc().year()`, rfc3164_decoder.rs:175);
        0 = the UTC year of the clock at each call."""
        self._check(self.L.fg_set_rfc3164_year(self.ctx, year), "fg_set_rfc3164_year")

    def set_tz_table(self, zones: dict[str, tuple[list[int], list[int]]]) -> None:
        """Replace the zone database: name -> (UTC transition seconds, len + 1 UTC offsets), as oracle/tzread.py yields."""
        names = sorted(zones)
        first = np.zeros(len(names) + 1, dtype=np.int32)
        starts, offs = [], []
        for k, nm in enumerate(names):
            tr, of = zones[nm]
            starts += [0] + [int(t) for t in tr]
            offs += [int(o) for o in of]
            first[k + 1] = len(offs)
        st = np.asarray(starts, dtype=np.int64)
        of = np.asarray(offs, dtype=np.int32)
        cn = (C.c_char_p * max(len(names), 1))(*[n.encode() for n in names])
        self._check(self.L.fg_set_tz_table(self.ctx, len(names), cn, _ptr(first), _ptr(st), _ptr(of)), "fg_set_tz_table")

    def close(self) -> None:
        if self._h:
            for p in self._pinned:
                self.L.fg_host_free(self.ctx, p)
            self._pinned.clear()
            self.H.fgh_decoder_free(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _check(self, rc: int, what: str) -> None:
        if rc != 0:
            raise RuntimeError(f"{what} failed ({rc}): {self.L.fg_last_error(self.ctx).decode()}")

    def host_alloc(self, nbytes: int, dtype=np.uint8) -> np.ndarray:
        """Pinned host array (what a batching splitter fills directly)."""
        p = C.c_void_p()
        self._check(self.L.fg_host_alloc(self.ctx, max(nbytes, 1), C.byref(p)), "fg_host_alloc")
        self._pinned.append(p)
        a = np.ctypeslib.as_array(C.cast(p, C.POINTER(C.c_uint8)), shape=(max(nbytes, 1),))[:nbytes]
        return a.view(dtype)

    def decode(self, data: np.ndarray, offsets: np.ndarray) -> BatchResult:
        assert data.dtype == np.uint8 and offsets.dtype == np.int32
        out = FgBatchOut()
        n = len(offsets) - 1
        self._keep = (data, offsets)
        self._check(self.L.fg_decode_batch(self.ctx, self.fmt, _ptr(data), _ptr(offsets), n, C.byref(out)), "fg_decode_batch")
        return BatchResult(out, self.fmt)

    def set_gelf_extra(self, extra: dict[str, str]) -> None:
        """output.gelf_extra of GelfEncoder::new (gelf_encoder.rs:29-48)."""
        self._check(self.L.fg_set_gelf_extra(self.ctx, *_extra_arrays(extra)), "fg_set_gelf_extra")

    def set_output_framing(self, framing: int) -> None:
        """output.framing of the fused calls (fg_set_output_framing): OUT_NONE, OUT_LINE ("\\n" after each record), OUT_NUL
        ("\\0" after each record) or OUT_SYSLEN ("{len + 1} " before, "\\n" after).  A rejected record stays empty, so the
        bytes of a fused call are the whole output stream of its batch."""
        self._check(self.L.fg_set_output_framing(self.ctx, framing), "fg_set_output_framing")

    def decode_encode_gelf(self, data: np.ndarray, offsets: np.ndarray, copy: bool = True):
        """decode + GelfEncoder::encode fused on the device, for a decoder of FMT_RFC5424, FMT_RFC3164, FMT_LTSV or
        FMT_GELF: (JSON bytes, int64 offsets[n+1], status uint8[n], kernel ms).  An RFC3164 record has no application_name,
        process_id or sd_id, "level" only when the line has a <PRI>, and always a "short_message" (possibly "").  An LTSV
        record has no application_name, process_id or sd_id, one "_" + name (+ type suffix) key per pair with typed
        values as JSON bools / numbers, and "-" as short_message without a `message` part; ltsv_stops() gives its
        "Missing value" lines.  A GELF record has no application_name, process_id or sd_id, "level" and
        "full_message" only when the object has them, one "_" + name key per other member (the name alone when it starts
        with "_"), strings re-escaped from their unescaped text, and gelf_now() as "timestamp" when the object has none.
        With copy=False the arrays are views of the context's pinned buffers (valid until the
        next call)."""
        return self._decode_encode("fg_decode_encode_gelf", data, offsets, copy)

    def set_ltsv_extra(self, extra: dict[str, str]) -> None:
        """output.ltsv_extra of LTSVEncoder::new (ltsv_encoder.rs:10-30); written in byte order of the keys."""
        self._check(self.L.fg_set_ltsv_extra(self.ctx, *_extra_arrays(extra)), "fg_set_ltsv_extra")

    def decode_encode_ltsv(self, data: np.ndarray, offsets: np.ndarray, copy: bool = True):
        """decode + LTSVEncoder::encode fused on the device (fg_decode_encode_ltsv), for the same four decoders as
        decode_encode_gelf and with the same results: (LTSV bytes, int64 offsets[n+1], status uint8[n], kernel ms).  A
        record is `key:value` fields separated by tabs in Record order: the SD pairs (names without their leading "_"),
        the extras, host, time (Rust's Display for f64), then message, full_message, level, facility, appname, procid and
        msgid where the Record has them."""
        return self._decode_encode("fg_decode_encode_ltsv", data, offsets, copy)

    def split_decode_encode_ltsv(self, stream: np.ndarray, framing: int = 0, copy: bool = True):
        """split_decode_encode_gelf with the LTSV encoder (fg_split_decode_encode_ltsv)."""
        return self._split_decode_encode("fg_split_decode_encode_ltsv", stream, framing, copy)

    def set_capnp_extra(self, extra: dict[str, str]) -> None:
        """output.capnp_extra of CapnpEncoder::new (capnp_encoder.rs:14-32); written in byte order of the keys."""
        self._check(self.L.fg_set_capnp_extra(self.ctx, *_extra_arrays(extra)), "fg_set_capnp_extra")

    def decode_encode_capnp(self, data: np.ndarray, offsets: np.ndarray, copy: bool = True):
        """decode + CapnpEncoder::encode fused on the device (fg_decode_encode_capnp), for the same four decoders as
        decode_encode_gelf and with the same results: (Cap'n Proto bytes, int64 offsets[n+1], status uint8[n], kernel ms).
        A record is the serialized message of record.capnp's Record: the segment table, then the segments' words.  The
        default output.framing of capnp is none ("noop")."""
        return self._decode_encode("fg_decode_encode_capnp", data, offsets, copy)

    def split_decode_encode_capnp(self, stream: np.ndarray, framing: int = 0, copy: bool = True):
        """split_decode_encode_gelf with the Cap'n Proto encoder (fg_split_decode_encode_capnp)."""
        return self._split_decode_encode("fg_split_decode_encode_capnp", stream, framing, copy)

    def set_passthrough_prefix(self, header: bytes) -> None:
        """The header of the following passthrough calls (output.syslog_prepend_timestamp, formatted by the caller), written
        as given; b"" clears it."""
        self._check(self.L.fg_set_passthrough_prefix(self.ctx, header, len(header)), "fg_set_passthrough_prefix")

    def decode_encode_passthrough(self, data: np.ndarray, offsets: np.ndarray, copy: bool = True):
        """decode + PassthroughEncoder::encode fused on the device (fg_decode_encode_passthrough), for the same four
        decoders as decode_encode_gelf and with the same results: (records, int64 offsets[n+1], status uint8[n], kernel ms).
        Record i is the header + Record.full_msg; a GELF object without full_message has status FG_EP_NO_RAW and no
        record.  The default output.framing of passthrough is none ("noop"), "line" for output.type = "debug"."""
        return self._decode_encode("fg_decode_encode_passthrough", data, offsets, copy)

    def split_decode_encode_passthrough(self, stream: np.ndarray, framing: int = 0, copy: bool = True):
        """split_decode_encode_gelf with the passthrough encoder (fg_split_decode_encode_passthrough)."""
        return self._split_decode_encode("fg_split_decode_encode_passthrough", stream, framing, copy)

    def _decode_encode(self, fn: str, data: np.ndarray, offsets: np.ndarray, copy: bool):
        assert data.dtype == np.uint8 and offsets.dtype == np.int32
        out = FgEncodedOut()
        n = len(offsets) - 1
        self._keep = (data, offsets)
        self._check(getattr(self.L, fn)(self.ctx, self.fmt, _ptr(data), _ptr(offsets), n, C.byref(out)), fn)
        self._last_encoded_n = n
        buf, offs, status = _encoded_views(out)
        if copy:
            return buf.tobytes(), offs.copy(), status.copy(), out.kernel_ms
        return buf, offs, status, out.kernel_ms

    def split_decode_encode_gelf(self, stream: np.ndarray, framing: int = 0, copy: bool = True):
        """Framing (0 = "line", 1 = "nul") + UTF-8 validation + decode (FMT_RFC5424, FMT_RFC3164, FMT_LTSV or FMT_GELF) + GelfEncoder::encode
        of a raw byte stream, all on the device: (JSON bytes, int64 offsets[n+1], status uint8[n], record starts
        int32[n+1] in `stream` with their terminators, kernel ms).  A record that is not UTF-8 has status 76
        ("Invalid UTF-8 input") and an empty JSON record.
        With copy=False the arrays are views of the context's pinned buffers (valid until the next call)."""
        return self._split_decode_encode("fg_split_decode_encode_gelf", stream, framing, copy)

    def _split_decode_encode(self, fn: str, stream: np.ndarray, framing: int, copy: bool):
        assert stream.dtype == np.uint8
        out = FgEncodedOut()
        lo = C.POINTER(C.c_int32)()
        self._keep = (stream,)
        self._check(getattr(self.L, fn)(self.ctx, self.fmt, framing, _ptr(stream), len(stream), C.byref(out), C.byref(lo)), fn)
        n = out.n
        self._last_encoded_n = n
        buf, offs, status = _encoded_views(out)
        lines = np.ctypeslib.as_array(lo, shape=(n + 1,))
        if copy:
            return buf.tobytes(), offs.copy(), status.copy(), lines.copy(), out.kernel_ms
        return buf, offs, status, lines, out.kernel_ms

    def ltsv_stops(self) -> np.ndarray:
        """After decode_encode_gelf / split_decode_encode_gelf on an LTSV decoder: int32[n], -1 where the decoder printed
        nothing, else the offset from the record's start up to which its parts were read (fg_encoded_ltsv_stops); every
        part before it without ':' printed "Missing value for name '<part>'"."""
        p = C.POINTER(C.c_int32)()
        self._check(self.L.fg_encoded_ltsv_stops(self.ctx, C.byref(p)), "fg_encoded_ltsv_stops")
        n = self._last_encoded_n
        return np.ctypeslib.as_array(p, shape=(n,)).copy() if n else np.zeros(0, np.int32)

    def gelf_now(self) -> float:
        """After decode_encode_gelf / split_decode_encode_gelf on a GELF decoder: the "timestamp" its records without one
        were given, the wall clock read once at the start of that call (fg_encoded_gelf_now)."""
        v = C.c_double()
        self._check(self.L.fg_encoded_gelf_now(self.ctx, C.byref(v)), "fg_encoded_gelf_now")
        return v.value

    def split_decode(self, stream: np.ndarray, framing: int | None = None) -> BatchResult:
        """Framing + UTF-8 validation + decode of a raw byte stream, all on the device: fg_split_decode (newline
        framing), or fg_split_decode_framed with `framing` 0 = "line", 1 = "nul".  The record starts, n + 1 int32, are at
        BatchResult.raw.line_offsets."""
        assert stream.dtype == np.uint8
        out = FgBatchOut()
        self._keep = (stream,)
        if framing is None:
            self._check(self.L.fg_split_decode(self.ctx, self.fmt, _ptr(stream), len(stream), C.byref(out)), "fg_split_decode")
        else:
            self._check(self.L.fg_split_decode_framed(self.ctx, self.fmt, framing, _ptr(stream), len(stream), C.byref(out)),
                        "fg_split_decode_framed")
        return BatchResult(out, self.fmt)

    def last_split_ms(self) -> float:
        return float(self.L.fg_last_split_ms(self.ctx))

    def upload(self, data: np.ndarray, offsets: np.ndarray) -> None:
        assert data.dtype == np.uint8 and offsets.dtype == np.int32
        self._check(self.L.fg_upload(self.ctx, _ptr(data), _ptr(offsets), len(offsets) - 1), "fg_upload")

    def parse_resident(self) -> float:
        ms = C.c_float()
        self._check(self.L.fg_parse_resident(self.ctx, self.fmt, C.byref(ms)), "fg_parse_resident")
        return ms.value

    def last_dominant_kernel_ms(self) -> float:
        """CUDA-event time of the dominant kernel alone inside the last parse_resident() step."""
        return float(self.L.fg_last_dominant_kernel_ms(self.ctx))

    def parse_resident_many(self, k: int) -> float:
        """k back-to-back passes over the resident batch, one host sync; returns the CUDA-event time of all k (ms)."""
        ms = C.c_float()
        self._check(self.L.fg_parse_resident_n(self.ctx, self.fmt, k, C.byref(ms)), "fg_parse_resident_n")
        return ms.value

    def download(self) -> BatchResult:
        out = FgBatchOut()
        self._check(self.L.fg_download(self.ctx, self.fmt, C.byref(out)), "fg_download")
        return BatchResult(out, self.fmt)

    def flush_l2(self) -> None:
        self._check(self.L.fg_flush_l2(self.ctx), "fg_flush_l2")

    def kernel_launches(self) -> int:
        return int(self.L.fg_kernel_launches(self.ctx))

    def dump(self, res: BatchResult, data: np.ndarray, offsets: np.ndarray, nthreads: int = 8, lo: int = 0,
             hi: int | None = None) -> tuple[bytes, np.ndarray]:
        """Materialise the Records of lines [lo, hi) of a decoded batch and render the canonical parity dump."""
        hi = res.n if hi is None else hi
        pb, po = C.c_void_p(), C.c_void_p()
        self.H.fgh_dump_range(self._h, C.byref(res.raw), _ptr(data), _ptr(offsets), lo, hi, nthreads, C.byref(pb), C.byref(po))
        return _take_dumps(pb, po, hi - lo)

    def split_dump(self, stream: np.ndarray, framing: int = 0) -> tuple[bytes, np.ndarray, np.ndarray, float]:
        """fg_split_decode_framed on a raw byte stream (framing 0 = "line", 1 = "nul"): (canonical dumps, dump offsets,
        record offsets int32[n+1], kernel ms)."""
        assert stream.dtype == np.uint8
        pb, po, pl = C.c_void_p(), C.c_void_p(), C.c_void_p()
        n, ms = C.c_int32(), C.c_float()
        err = C.create_string_buffer(512)
        rc = self.H.fgh_split_dump(self._h, framing, _ptr(stream), len(stream), C.byref(pb), C.byref(po), C.byref(pl), C.byref(n), C.byref(ms), err, 512)
        if rc != 0:
            raise RuntimeError(err.value.decode())
        try:
            lines = np.ctypeslib.as_array(C.cast(pl, C.POINTER(C.c_int32)), shape=(n.value + 1,)).copy()
        finally:
            self.H.fgh_free(pl)
        return *_take_dumps(pb, po, n.value), lines, ms.value

    def materialize_seconds(self, res: BatchResult, data: np.ndarray, offsets: np.ndarray, nthreads: int = 1) -> float:
        return float(self.H.fgh_materialize_bench(self._h, C.byref(res.raw), _ptr(data), _ptr(offsets), nthreads))


def dump_records(fmt: int, out: FgBatchOut, data: np.ndarray, offsets: np.ndarray,
                 ltsv_suffix: list | None = None) -> tuple[bytes, np.ndarray]:
    """The product's Record materialiser + canonical dump over bare result arrays (no device, no context).
    ltsv_suffix: 5 entries indexed by fg_ltsv_type (bytes or None)."""
    H = load_host()
    pb, po = C.c_void_p(), C.c_void_p()
    suf = None
    if ltsv_suffix is not None:
        suf = (C.c_char_p * 5)(*[s if s is None else bytes(s) for s in ltsv_suffix])
    H.fgh_dump_records(fmt, C.byref(out), _ptr(data), _ptr(offsets), suf, C.byref(pb), C.byref(po))
    return _take_dumps(pb, po, out.n)


def tz_lookup(name: str, local: int, tzdir: str | None = None):
    """Host-side query of the zone database a context loads (fg_tz_lookup): UTC offset of `name` at the local second, or None."""
    L = load_cuda()
    off = C.c_int32()
    rc = L.fg_tz_lookup(tzdir.encode() if tzdir else None, name.encode(), local, C.byref(off))
    if rc < 0:
        raise RuntimeError("no zone database")
    return int(off.value) if rc == 1 else None


def tz_count(tzdir: str | None = None) -> int:
    return int(load_cuda().fg_tz_count(tzdir.encode() if tzdir else None))


def shard_by_bytes(offsets: np.ndarray, G: int) -> np.ndarray:
    """SURVEY.md §8(e): contiguous line ranges balanced by bytes; returns bounds int32[G+1]."""
    assert offsets.dtype == np.int32
    bounds = np.zeros(G + 1, dtype=np.int32)
    load_host().fgh_shard_by_bytes(_ptr(offsets), len(offsets) - 1, G, _ptr(bounds))
    return bounds


def multi_gpu_decode_dump(fmt: int, devices: list[int], data: np.ndarray, offsets: np.ndarray) -> tuple[bytes, np.ndarray]:
    """Decode one batch on several GPUs (one host thread + context per device) and return the canonical dumps."""
    H = load_host()
    dev = np.asarray(devices, dtype=np.int32)
    pb, po = C.c_void_p(), C.c_void_p()
    err = C.create_string_buffer(512)
    n = len(offsets) - 1
    rc = H.fgh_multi_decode_dump(fmt, _ptr(dev), len(devices), int(offsets[-1]) + (1 << 20), n + 1024, _ptr(data), _ptr(offsets), n,
                                 C.byref(pb), C.byref(po), err, 512)
    if rc != 0:
        raise RuntimeError(err.value.decode())
    return _take_dumps(pb, po, n)


def clone_decode_threads(fmt: int, lines: list[bytes], nthreads: int = 2, device: int = 0) -> list[bytes]:
    """Decoder::clone_boxed() + concurrent Decoder::decode(line) from `nthreads` host threads; canonical dump per line."""
    H = load_host()
    offs = np.zeros(len(lines) + 1, dtype=np.int32)
    np.cumsum([len(x) for x in lines], out=offs[1:])
    data = np.frombuffer(b"".join(lines) or b"\0", dtype=np.uint8).copy()
    pb, po = C.c_void_p(), C.c_void_p()
    err = C.create_string_buffer(512)
    rc = H.fgh_clone_decode_threads(fmt, device, _ptr(data), _ptr(offs), len(lines), nthreads, C.byref(pb), C.byref(po), err, 512)
    if rc != 0:
        raise RuntimeError(err.value.decode())
    buf, o = _take_dumps(pb, po, len(lines))
    return [buf[o[i]:o[i + 1]] for i in range(len(lines))]


def splitter_run_gelf(dec: "BatchDecoder", text: bytes, extra: dict[str, str] | None = None, max_lines: int = 1 << 16,
                      max_bytes: int = 16 << 20, framing: int = 0, stdout: bool = False) -> tuple[bytes, ...]:
    """BatchingLineSplitter (framing 0), BatchingNulSplitter (framing 1) or BatchingSyslenSplitter (framing 2: records
    framed on the host and batched by RecordBatcher) with input.format = rfc5424, rfc3164, ltsv or gelf (the decoder's format)
    and output.format = gelf (decode and encode fused on the GPU, framing too for 0 and 1): returns (JSON records
    separated by newlines, stderr text), and with stdout=True also the stdout text (LTSV's "Missing value" lines)."""
    H = load_host()
    n_extra, keys, vals = _extra_arrays(extra)
    out = _run_splitter(lambda o: H.fgh_splitter_run_gelf(dec._h, text, len(text), max_lines, max_bytes, n_extra, keys, vals,
                                                          *o[:4], framing, *o[4:]))
    return out if stdout else out[:2]


def splitter_run_gelf_framed(dec: "BatchDecoder", text: bytes, out_framing: int, extra: dict[str, str] | None = None,
                             max_lines: int = 1 << 16, max_bytes: int = 16 << 20, framing: int = 0) -> tuple[bytes, bytes, bytes]:
    """splitter_run_gelf with output.framing applied on the device (OUT_NONE, OUT_LINE, OUT_NUL or OUT_SYSLEN): returns
    (the output stream exactly as the splitter sent it, stderr text, stdout text)."""
    H = load_host()
    n_extra, keys, vals = _extra_arrays(extra)
    return _run_splitter(lambda o: H.fgh_splitter_run_gelf_framed(dec._h, text, len(text), max_lines, max_bytes, n_extra, keys,
                                                                  vals, framing, out_framing, *o))


def splitter_run_ltsv_framed(dec: "BatchDecoder", text: bytes, out_framing: int, extra: dict[str, str] | None = None,
                             max_lines: int = 1 << 16, max_bytes: int = 16 << 20, framing: int = 0) -> tuple[bytes, bytes, bytes]:
    """splitter_run_gelf_framed with output.format = "ltsv" (CudaLtsvEncoder, output.ltsv_extra = extra): returns (the
    output stream exactly as the splitter sent it, stderr text, stdout text)."""
    H = load_host()
    n_extra, keys, vals = _extra_arrays(extra)
    return _run_splitter(lambda o: H.fgh_splitter_run_ltsv_framed(dec._h, text, len(text), max_lines, max_bytes, n_extra, keys,
                                                                  vals, framing, out_framing, *o))


def splitter_run_capnp_framed(dec: "BatchDecoder", text: bytes, out_framing: int = 0, extra: dict[str, str] | None = None,
                              max_lines: int = 1 << 16, max_bytes: int = 16 << 20, framing: int = 0) -> tuple[bytes, bytes, bytes]:
    """splitter_run_gelf_framed with output.format = "capnp" (CudaCapnpEncoder, output.capnp_extra = extra; output.framing
    defaults to none, the reference's "noop" for capnp): returns (the output stream exactly as the splitter sent it, stderr
    text, stdout text)."""
    H = load_host()
    n_extra, keys, vals = _extra_arrays(extra)
    return _run_splitter(lambda o: H.fgh_splitter_run_capnp_framed(dec._h, text, len(text), max_lines, max_bytes, n_extra, keys,
                                                                   vals, framing, out_framing, *o))


def splitter_run_passthrough_framed(dec: "BatchDecoder", text: bytes, out_framing: int = 0, header: bytes | None = None,
                                    max_lines: int = 1 << 16, max_bytes: int = 16 << 20, framing: int = 0) -> tuple[bytes, bytes, bytes]:
    """splitter_run_gelf_framed with output.format = "passthrough" (CudaPassthroughEncoder, whose header source gives
    `header` for every device call, none when None; output.framing defaults to none, the reference's "noop"): returns (the
    output stream exactly as the splitter sent it, stderr text, stdout text)."""
    H = load_host()
    return _run_splitter(lambda o: H.fgh_splitter_run_passthrough_framed(dec._h, text, len(text), max_lines, max_bytes, header,
                                                                         len(header or b""), framing, out_framing, *o))


def splitter_run(dec: "BatchDecoder", text: bytes, max_lines: int = 1 << 16, max_bytes: int = 16 << 20,
                 framing: int = 0) -> tuple[bytes, bytes, bytes]:
    """Batching splitter over `text` (the stdin of config #1); framing 0 = "line", 1 = "nul", 2 = "syslen" (input.framing):
    returns (records, stderr, stdout)."""
    H = load_host()
    return _run_splitter(lambda o: H.fgh_splitter_run(dec._h, framing, text, len(text), max_lines, max_bytes, *o))
