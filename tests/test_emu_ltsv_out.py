"""CPU checks of the LTSV encoder's text: Rust's Display for f64 as the device formats it (fg_ftoa.cuh, Schubfach with the
126-bit table of fg_ftoa_table.inc) against its restatement over Python's repr (tests/ltsv_oracle.py), the key / value
replacements of LTSVString::insert (fg_ltsv_text.cuh), and the restated encoder pinned to the reference's own tests.
Both product headers are compiled with g++ (tests/emu/emu_ltsv_text.cpp).  No GPU needed."""
import ctypes as C
import json
import math
import struct
import subprocess
from pathlib import Path

import numpy as np
import pytest

import ltsv_oracle as LO

HERE = Path(__file__).resolve().parent


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    so = tmp_path_factory.mktemp("emu_ltsv_text") / "libfg_emu_ltsv_text.so"
    subprocess.run(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-Wno-unknown-pragmas", "-o", str(so),
                    str(HERE / "emu" / "emu_ltsv_text.cpp")], check=True)
    L = C.CDLL(str(so))
    L.emu_f64_display.restype = C.c_longlong
    L.emu_f64_display.argtypes = [C.c_void_p, C.c_longlong, C.c_void_p, C.c_longlong, C.c_void_p]
    L.emu_ltsv_escape.argtypes = [C.c_char_p, C.c_int, C.c_int, C.c_void_p]
    return L


def display(emu, values) -> list[str]:
    v = np.ascontiguousarray(values, dtype=np.float64)
    out = np.zeros(len(v) * 340 + 16, np.uint8)
    lens = np.zeros(len(v), np.int32)
    n = emu.emu_f64_display(v.ctypes.data, len(v), out.ctypes.data, len(out), lens.ctypes.data)
    assert n >= 0
    text = out[:n].tobytes().decode()
    ends = np.cumsum(lens)
    return [text[e - l:e] for e, l in zip(ends.tolist(), lens.tolist())]


def check(emu, values):
    got = display(emu, values)
    for x, g in zip(values, got):
        assert g == LO.rust_f64(float(x)), (repr(float(x)), g, LO.rust_f64(float(x)))


def test_special_values_and_layout(emu):
    cases = [(0.0, "0"), (-0.0, "-0"), (math.inf, "inf"), (-math.inf, "-inf"), (1.0, "1"), (1e21, "1000000000000000000000"),
             (1e-7, "0.0000001"), (5e-324, "0." + "0" * 323 + "5"), (1438854924.123, "1438854924.123"), (-2.5, "-2.5"),
             (1.7976931348623157e308, "17976931348623157" + "0" * 292)]
    assert display(emu, [v for v, _ in cases]) == [t for _, t in cases]
    assert display(emu, [math.nan]) == ["NaN"]


def test_powers_of_ten_and_two(emu):
    check(emu, [10.0 ** k for k in range(-323, 309)] + [2.0 ** k for k in range(-1074, 1024)] +
          [-(2.0 ** k) for k in range(-1074, 1024, 7)])


def test_timestamps(emu):
    rng = np.random.default_rng(7)
    secs = rng.integers(0, 4_000_000_000, 100_000)
    check(emu, (secs + rng.integers(0, 1_000_000, 100_000) / 1e6).tolist() + (secs + np.round(rng.random(100_000), 3)).tolist())


def test_where_grisu2_is_not_shortest(emu, oracle):
    """values whose serde_json (Grisu2, fg_dtoa.cuh) text has more digits than the shortest: found, then checked"""
    rng = np.random.default_rng(11)
    vals = rng.integers(0, 2 ** 64, 200_000, dtype=np.uint64).view(np.float64)
    vals = [float(v) for v in vals if math.isfinite(v) and v != 0][:20_000]
    longer = []
    for v in vals:
        g = oracle.format_f64(v)
        mant = g.split("e")[0].replace("-", "").replace(".", "").strip("0")
        if len(mant) > len(repr(v).split("e")[0].replace("-", "").replace(".", "").strip("0")):
            longer.append(v)
    assert longer, "no value where Grisu2 is longer than the shortest"
    check(emu, longer)


def test_random_bit_patterns(emu):
    rng = np.random.default_rng(3)
    for seed in range(4):
        bits = np.random.default_rng(seed).integers(0, 2 ** 64, 300_000, dtype=np.uint64)
        bits[:5000] &= np.uint64(0x800FFFFFFFFFFFFF)  # subnormals
        check(emu, bits.view(np.float64).tolist())
    assert rng is not None


@pytest.mark.parametrize("key", [0, 1])
def test_escapes(emu, key):
    rng = np.random.default_rng(5 + key)
    alphabet = np.frombuffer(b"ab:\t\n\r \x00\xc3\xa9_", np.uint8)
    for n in list(range(0, 12)) + [37, 64, 1001]:
        for _ in range(30):
            s = alphabet[rng.integers(0, len(alphabet), n)].tobytes()
            out = C.create_string_buffer(max(n, 1))
            emu.emu_ltsv_escape(s, n, key, out)
            assert out.raw[:n] == (LO.esc_key(s) if key else LO.esc_val(s)), s


def test_reference_encoder_tests():
    doc = json.loads((HERE / "golden" / "ltsv_encoder_tests.json").read_text())
    for case in doc["cases"]:
        r = dict(case["record"])
        for k in ("host", "app", "proc", "msgid", "msg", "full"):
            r[k] = r[k].encode()
        r["sd"] = None if r["sd"] is None else [[(k.encode(), v.encode()) for k, v in sd] for sd in r["sd"]]
        assert LO.encode(r, []).decode() == case["expected"], case["source"]


def test_oracle_records_from_dumps(oracle):
    """the restated encoder over the oracle's decoded Records: names lose one '_', extras in byte order of their keys
    as given ("_z" before "a")"""
    d, o = oracle.pack([b'<23>1 2015-08-05T15:53:45.637824Z h app 69 42 [o@1 _k="v\tw" a:b="c"] msg',
                        b'{"host":"","short_message":"m","_n":null,"__x":1.5e300,"timestamp":0.1}'])
    r5 = LO.decode_encode_ltsv(oracle, 0, d[:o[1]].copy(), o[:2].copy(), extra={"_z": "1", "a": "t\tx"})
    assert r5 == [b"_k:v w\ta_b:c\tz:1\ta:t x\thost:h\ttime:1438790025.637824\tmessage:msg\tfull_message:"
                  + bytes(d[:o[1]]).replace(b"\t", b" ") + b"\tlevel:7\tfacility:2\tappname:app\tprocid:69\tmsgid:42"]
    g = LO.decode_encode_ltsv(oracle, 2, (d[o[1]:]).copy(), (o[1:] - o[1]).astype(np.int32))
    assert g == [b"_x:15" + b"0" * 299 + b"\tn:\thost:\ttime:0.1\tmessage:m"]
    assert struct.calcsize("<d") == 8
