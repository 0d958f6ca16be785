"""CPU check of the fused GELF encoder's string re-encoding: json_transcode_step (fg_gelf.cuh, the decoder's KeyIter
unescape + serde_json's escape), compiled with g++ (tests/emu/emu_json.cpp) and driven over whole string bodies, against
the oracle's decode + encode of the same body as a short_message: every non-surrogate \\uXXXX, a sample of surrogate
pairs, every short escape and the newline-retry forms.  No GPU needed."""
import ctypes as C
import subprocess
from pathlib import Path

import numpy as np
import pytest

HERE = Path(__file__).resolve().parent
GELF = 2


@pytest.fixture(scope="module")
def transcode(tmp_path_factory):
    so = tmp_path_factory.mktemp("emu_json") / "libfg_emu_json.so"
    subprocess.run(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-Wno-unknown-pragmas", "-o", str(so),
                    str(HERE / "emu" / "emu_json.cpp")], check=True)
    L = C.CDLL(str(so))
    L.emu_json_transcode.argtypes = [C.c_char_p, C.c_int, C.c_int, C.c_void_p, C.c_int]

    def run(body: bytes, mode2: bool) -> bytes:
        out = C.create_string_buffer(4 * len(body) + 16)
        n = L.emu_json_transcode(body, len(body), 1 if mode2 else 0, out, len(out))
        assert n >= 0
        return out.raw[:n]
    return run


def oracle_texts(oracle, bodies: list[bytes]) -> list[bytes]:
    """serde_json's text of each body's unescaped string: the short_message of {"host":"h","short_message":"<body>"}"""
    lines = [b'{"host":"h","short_message":"' + b + b'","timestamp":1}' for b in bodies]
    d, o = oracle.pack(lines)
    buf, offs = oracle.decode_encode_gelf(GELF, d, o, nthreads=8)
    out = []
    for i in range(len(lines)):
        rec = buf[offs[i]:offs[i + 1]]
        assert rec, lines[i]
        a = rec.index(b'"short_message":"') + len(b'"short_message":"')
        out.append(rec[a:rec.rindex(b'","timestamp":')])
    return out


def check(transcode, oracle, bodies, mode2=False):
    want = oracle_texts(oracle, bodies)
    for b, w in zip(bodies, want):
        assert transcode(b, mode2) == w, (b, transcode(b, mode2), w)


def test_every_bmp_escape(transcode, oracle):
    cps = [c for c in range(0x10000) if not 0xD800 <= c <= 0xDFFF]
    for k in range(0, len(cps), 4096):
        chunk = cps[k:k + 4096]
        check(transcode, oracle, [b"\\u%04x" % c for c in chunk] + [b"ab\\u%04Xcd\\/" % c for c in chunk[::7]])


def test_surrogate_pairs(transcode, oracle):
    rng = np.random.default_rng(3)
    hi = [0xD800, 0xDBFF] + [int(x) for x in rng.integers(0xD800, 0xDC00, 300)]
    lo = [0xDC00, 0xDFFF] + [int(x) for x in rng.integers(0xDC00, 0xE000, 300)]
    check(transcode, oracle, [b"x\\u%04x\\u%04X" % (h, l) for h, l in zip(hi, lo)])


def test_short_escapes_and_runs(transcode, oracle):
    short = [b"\\\"", b"\\\\", b"\\/", b"\\b", b"\\f", b"\\n", b"\\r", b"\\t"]
    bodies = short + [b"abcdefgh" + e + b"ijk" + e for e in short] + [b"".join(short) * 3, b"plain text only", b"",
                                                                      "é日本\U0001F680".encode(), b"a\\u00e9bcd\\u0000efgh"]
    check(transcode, oracle, bodies)


def test_retry_lines(transcode, oracle):
    """mode2: a raw LF is the `\\n` escape of the retry text, and `\\` + LF becomes `\\\\n`"""
    bodies = [b"a\nb", b"\n", b"\\\n", b"x\\\ny\n\\u00e9\n", b"abcd\nefgh\\\\\n", b"\\\"\n\\/"]
    lines = [b'{"host":"h\n","short_message":"' + b + b'","timestamp":1}' for b in bodies]
    d, o = oracle.pack(lines)
    buf, offs = oracle.decode_encode_gelf(GELF, d, o, nthreads=2)
    for i, b in enumerate(bodies):
        rec = buf[offs[i]:offs[i + 1]]
        assert rec, lines[i]
        a = rec.index(b'"short_message":"') + len(b'"short_message":"')
        assert transcode(b, True) == rec[a:rec.rindex(b'","timestamp":')], b
