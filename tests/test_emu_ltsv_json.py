"""CPU check of the fused LTSV encoder's GELF string path: json_unescape_step (fg_gelf.cuh) and ltsv_escape4
(fg_ltsv_text.cuh), compiled with g++ (tests/emu/emu_ltsv_json.cpp) and driven over whole JSON string bodies the way
run_ltsv does, against the oracle's GELF decode encoded by LTSVEncoder::encode restated (tests/ltsv_oracle.py): every
non-surrogate \\uXXXX alone and at each offset mod 4 of the four-byte word, the bounds and a sample of surrogate pairs,
every short escape in runs, raw UTF-8 and the newline-retry forms, as a value (short_message) and as a key (a member
name, its one leading '_' stripped, whether plain or spelled \\u005f).  No GPU needed."""
import ctypes as C
import subprocess
from pathlib import Path

import numpy as np
import pytest

import ltsv_oracle as LO

HERE = Path(__file__).resolve().parent
GELF = 2
SHORT = [b"\\\"", b"\\\\", b"\\/", b"\\b", b"\\f", b"\\n", b"\\r", b"\\t"]
CPS = [c for c in range(0x10000) if not 0xD800 <= c <= 0xDFFF]


@pytest.fixture(scope="module")
def unescape(tmp_path_factory):
    so = tmp_path_factory.mktemp("emu_ltsv_json") / "libfg_emu_ltsv_json.so"
    subprocess.run(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-Wno-unknown-pragmas", "-o", str(so),
                    str(HERE / "emu" / "emu_ltsv_json.cpp")], check=True)
    L = C.CDLL(str(so))
    L.emu_ltsv_json.argtypes = [C.c_char_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_int]

    def run(body: bytes, mode2: bool, key: bool) -> bytes:
        out = C.create_string_buffer(4 * len(body) + 16)
        n = L.emu_ltsv_json(body, len(body), 1 if mode2 else 0, 1 if key else 0, out, len(out))
        assert n >= 0
        return out.raw[:n]
    return run


def _records(oracle, lines):
    d, o = oracle.pack(lines)
    return LO.decode_encode_ltsv(oracle, GELF, d, o, nthreads=8)


def value_texts(oracle, bodies, host=b"h"):
    """the message field of {"host":<host>,"short_message":"<body>"} through the oracle's decoder and LTSV encoder"""
    recs = _records(oracle, [b'{"host":"' + host + b'","short_message":"' + b + b'","timestamp":1}' for b in bodies])
    out = []
    for b, rec in zip(bodies, recs):
        assert rec, b
        msg = [f for f in rec.split(b"\t") if f.startswith(b"message:")]
        assert len(msg) == 1, rec
        out.append(msg[0][len(b"message:"):])
    return out


def key_texts(oracle, bodies, host=b"h"):
    """the key the encoder writes for the member "<body>":"v" (the record's first field); None where the oracle's
    decoder rejects the line"""
    recs = _records(oracle, [b'{"host":"' + host + b'","short_message":"m","' + b + b'":"v","timestamp":1}' for b in bodies])
    out = []
    for rec in recs:
        if not rec:
            out.append(None)
            continue
        assert rec.count(b":v\thost:") == 1, rec
        out.append(rec[:rec.index(b":v\thost:")])
    return out


def _strip_underscore(body: bytes) -> bytes:
    """the member name the encoder reads (load_pair_gelf): one leading '_', a raw byte or the escape that spells it, off"""
    if body.startswith(b"_"):
        return body[1:]
    if body[:6].lower() == b"\\u005f":
        return body[6:]
    return body


def check_values(unescape, oracle, bodies, mode2=False, host=b"h"):
    for b, w in zip(bodies, value_texts(oracle, bodies, host)):
        got = unescape(b, mode2, False)
        assert got == w, (b, got, w)


def check_keys(unescape, oracle, bodies, mode2=False, host=b"h"):
    want = key_texts(oracle, bodies, host)
    assert sum(w is None for w in want) <= len(bodies) // 100, "the oracle rejects too many of the key lines"
    for b, w in zip(bodies, want):
        if w is None:
            continue
        got = unescape(_strip_underscore(b), mode2, True)
        assert got == w, (b, got, w)


def _around(c: int, lead: int) -> bytes:
    """\\uXXXX after `lead` plain bytes, so that its backslash falls on word offset lead mod 4, then plain bytes"""
    return b"ab:"[:lead] + b"\\u%04x" % c + b"xyz"


def test_every_bmp_escape_as_value(unescape, oracle):
    for k in range(0, len(CPS), 8192):
        chunk = CPS[k:k + 8192]
        check_values(unescape, oracle, [b"\\u%04X" % c for c in chunk] + [_around(c, j) for c in chunk for j in range(4)])


def test_every_bmp_escape_as_key(unescape, oracle):
    for k in range(0, len(CPS), 8192):
        chunk = CPS[k:k + 8192]
        check_keys(unescape, oracle, [b"\\u%04x" % c for c in chunk] + [_around(c, j) for c in chunk[::5] for j in range(4)])


def _pairs():
    rng = np.random.default_rng(29)
    hi = [0xD800, 0xDBFF] + [int(x) for x in rng.integers(0xD800, 0xDC00, 300)]
    lo = [0xDC00, 0xDFFF] + [int(x) for x in rng.integers(0xDC00, 0xE000, 300)]
    return [b"ab:"[:j % 4] + b"\\u%04x\\u%04X" % (h, l) + b"\\t" * (j % 3) for j, (h, l) in enumerate(zip(hi, lo))]


def test_surrogate_pairs(unescape, oracle):
    bodies = _pairs()
    check_values(unescape, oracle, bodies)
    check_keys(unescape, oracle, bodies)


def _short_bodies():
    runs = [b"".join(SHORT) * 3, b"\\t\\n" * 5, b"\\\\" * 7, b"\\\\\\\"" * 3]
    return SHORT + [b"abcdefgh"[:j] + e + b"ijk:" + e for e in SHORT for j in range(5)] + runs + [
        b"plain text only", b"", b"a:b", "é日本\U0001F680".encode(), "x:é\t"[:3].encode() + "日本:\U0001F680ab".encode(),
        b"a\\u00e9bcd\\u0000efgh", b"\\u0009\\u000a\\u003a\\u003A:", b"tab\\tcolon:nl\\n"]


def test_short_escapes_and_raw_utf8(unescape, oracle):
    bodies = _short_bodies()
    check_values(unescape, oracle, bodies)
    check_keys(unescape, oracle, [b for b in bodies if b])


def test_leading_underscore_keys(unescape, oracle):
    """a member name whose '_' is plain or the escape \\u005f: one '_' is stripped, a second one stays"""
    bodies = [b"_x", b"\\u005fx", b"\\u005Fx", b"__x", b"\\u005f_x", b"_\\u005fx", b"\\u005f\\u005f", b"_:", b"\\u005f\\t:",
              b"_\\u00e9", b"\\u005f\\ud83d\\ude80", b"_abcd\\\\efgh", b"\\u005f" + b"".join(SHORT)]
    check_keys(unescape, oracle, bodies)


RETRY = [b"a\nb", b"\n", b"\\\n", b"x\\\ny\n\\u00e9\n", b"abcd\nefgh\\\\\n", b"\\\"\n\\/", b"abc\\\n", b"\n\n\n\n\\\n\\\n",
         b"ab:\\t\\u003a\n"]


def test_retry_lines(unescape, oracle):
    """mode2 (a raw LF in the line): a raw LF stays LF (then ' '), and `\\` + LF is the two bytes `\\` 'n'"""
    check_values(unescape, oracle, RETRY, mode2=True, host=b"h\n")
    check_keys(unescape, oracle, RETRY + [b"_a\nb", b"\\u005f\\\n"], mode2=True, host=b"h\n")
