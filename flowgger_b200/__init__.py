"""flowgger_b200 — H100-native batched log-line decoder (RFC5424 / LTSV / GELF bytes -> Record).

Drop-in for flowgger's Decoder stage (`flowgger src/flowgger/decoder/mod.rs:44-46`): the
product is the C-ABI shared library `lib/libflowgger_cuda.so` (see `include/flowgger_cuda.h`); this
Python package is a thin ctypes binding over it used by the tests and `bench.py`.  There is no CPU
fallback: importing works anywhere, but constructing a decoder needs the built library and a GPU.
"""
from .native import (  # noqa: F401
    FMT_GELF,
    FMT_LTSV,
    FMT_RFC3164,
    FMT_RFC5424,
    OUT_LINE,
    OUT_NONE,
    OUT_NUL,
    OUT_SYSLEN,
    BatchDecoder,
    BatchResult,
    NativeLibraryMissing,
    build_info,
    clone_decode_threads,
    cuda_lib_path,
    dump_records,
    error_string,
    generate,
    load_cuda,
    load_gen,
    load_host,
    multi_gpu_decode_dump,
    shard_by_bytes,
    splitter_run,
    splitter_run_capnp_framed,
    splitter_run_gelf,
    splitter_run_gelf_framed,
    splitter_run_ltsv_framed,
    splitter_run_passthrough_framed,
    tz_count,
    tz_lookup,
)

__all__ = [
    "FMT_RFC5424", "FMT_LTSV", "FMT_GELF", "FMT_RFC3164", "BatchDecoder", "BatchResult", "NativeLibraryMissing",
    "build_info", "cuda_lib_path", "error_string", "generate", "load_cuda", "load_gen", "load_host",
]
