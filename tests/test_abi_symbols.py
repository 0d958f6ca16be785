"""The C-ABI library loads on a CPU-only box and exports every symbol include/flowgger_cuda.h declares.
No compute call is made here (there is no GPU and there is no CPU fallback)."""
import ctypes
import re
from pathlib import Path

REPO = Path(__file__).resolve().parent.parent


def declared_functions():
    text = (REPO / "include" / "flowgger_cuda.h").read_text()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    text = re.sub(r"static inline[^{]*\{.*?\n\}", "", text, flags=re.S)  # header-only span helpers (fg_row5424_*) are not exports
    return sorted(set(re.findall(r"\b(fg_[a-z0-9_]+)\s*\(", text)))


def test_header_symbols_exported(native):
    lib = native.load_cuda()
    names = declared_functions()
    assert len(names) >= 14
    for n in names:
        assert hasattr(lib, n), f"{n} declared in flowgger_cuda.h but not exported"


def test_error_strings_match_reference_text(native):
    # every status maps to the exact &'static str of the reference decoders (cited in fg_abi.cu)
    es = {native.error_string(0, s) for s in range(1, native.load_cuda().fg_error_count())} - {None}
    for must in ["Unsupported BOM", "The priority should be inside brackets", "Invalid priority", "Missing version",
                 "Unsupported version", "Missing timestamp",
                 "Unable to parse the date from RFC3339 to Unix time in RFC5424 decoder", "Missing hostname",
                 "Missing application name", "Missing process id", "Missing message id", "Missing message data",
                 "Missing log message", "Malformated RFC5424 message", "Missing structured data",
                 "Format error in the structured data", "Missing ] after structured data",
                 "Unable to parse the English to Unix timestamp in LTSV decoder", "Invalid severity level",
                 "Severity level should be <= 7", "Type error; boolean was expected", "Type error; f64 was expected",
                 "Type error; i64 was expected", "Type error; u64 was expected",
                 "Invalid GELF input, unable to parse as a JSON object", "Empty GELF input", "Invalid GELF timestamp",
                 "GELF host name must be a string", "GELF short message must be a string",
                 "GELF full message must be a string", "GELF version must be a string", "Unsupported GELF version",
                 "Invalid severity level (too high)", "Invalid value type in structured data",
                 "Malformed RFC3164 event: Invalid priority", "Malformed RFC3164 event: Invalid timestamp or hostname",
                 "Invalid time format", "Unable to parse RFC3164 date with year", "Unable to parse the date in RFC3164 decoder"]:
        assert must in es, must
    assert native.error_string(0, 0) is None


def test_reference_strings_present_in_reference_sources():
    """Guard against typos: each error string must occur verbatim in a string literal of the reference decoder and
    line-splitter sources (stored in tests/golden/reference_strings.json)."""
    import json
    import flowgger_b200 as fb
    golden = json.loads((REPO / "tests" / "golden" / "reference_strings.json").read_text())["literals"]
    assert "src/flowgger/splitter/line_splitter.rs" in golden  # "Invalid UTF-8 input"
    literals = [s for per_file in golden.values() for s in per_file]
    for s in range(1, fb.load_cuda().fg_error_count()):
        e = fb.error_string(0, s)
        if e and not e.startswith("(the reference panics here"):  # FG_E3_PANIC is this repo's name for a reference panic
            assert any(e in lit for lit in literals), e


def test_no_cpu_fallback_without_gpu(native):
    """On a box without a GPU the decoder must refuse to exist (fail loudly), never parse on the CPU."""
    import torch
    if torch.cuda.is_available():
        return
    import pytest
    with pytest.raises(RuntimeError, match="no CUDA device|fg_create"):
        native.BatchDecoder(native.FMT_RFC5424)


def test_build_info_names_sm90a(native):
    """The build string names sm_90a, and every device image embedded in the library is an sm_90a cubin (no other
    architecture, no PTX to JIT)."""
    import subprocess
    from flowgger_b200 import build as fb_build
    assert "sm_90a" in native.build_info()
    cuobjdump = str(Path(fb_build.NVCC).parent / "cuobjdump")
    lib = str(native.cuda_lib_path())
    elves = re.findall(r"\.(sm_\w+)\.cubin", subprocess.run([cuobjdump, "--list-elf", lib], capture_output=True, text=True,
                                                            check=True).stdout)
    assert elves and set(elves) == {"sm_90a"}, elves
    ptx = subprocess.run([cuobjdump, "--list-ptx", lib], capture_output=True, text=True, check=True).stdout
    assert "PTX file" not in ptx, ptx


def test_generator_is_deterministic(native):
    b1, o1 = native.generate(native.FMT_RFC5424, 5424, 2000)
    b2, o2 = native.generate(native.FMT_RFC5424, 5424, 2000, nthreads=3)
    assert (b1 == b2).all() and (o1 == o2).all()
    b3, o3 = native.generate(native.FMT_RFC5424, 5424, 1000, first_index=1000)
    assert bytes(b1[o1[1000]:]) == bytes(b3)
