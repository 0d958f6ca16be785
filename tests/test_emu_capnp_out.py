"""CPU checks of the Cap'n Proto encoder's layout: the device's allocator and pointer words (fg_capnp_layout.cuh, compiled
with g++ by tests/emu/emu_capnp.cpp) place every object of a message where the restated encoder (tests/capnp_oracle.py)
does and point to it with the same words, and the restated encoder is pinned to the reference's three tests and read
back by the wire-format reader.  Records cover the NUL / pad boundary of texts, messages of 1022..1026 words, objects
that back-fill segment 0 after a large one went to a new segment, extras across the segment boundary, 0, 1 and 1000
pairs and every union member.  The model of the encoder's segment list (tests/capnp_out_edges.py) joins to the
oracle's message on the random records and on every window line, whose coverage of the window boundaries is checked
here.  No GPU needed."""
import ctypes as C
import json
import random
import struct
import subprocess
from pathlib import Path

import numpy as np
import pytest

import capnp_oracle as O
import capnp_out_edges as CE

HERE = Path(__file__).resolve().parent


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    so = tmp_path_factory.mktemp("emu_capnp") / "libfg_emu_capnp.so"
    subprocess.run(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-Wno-unknown-pragmas", "-o", str(so),
                    str(HERE / "emu" / "emu_capnp.cpp")], check=True)
    L = C.CDLL(str(so))
    L.emu_capnp_layout.argtypes = [C.c_int] + [C.c_void_p] * 12
    L.emu_capnp_pairs_tag.restype = C.c_ulonglong
    L.emu_capnp_pairs_tag.argtypes = [C.c_uint32]
    return L


def f64(x: float) -> int:
    return struct.unpack("<Q", struct.pack("<d", x))[0]


def record(host=b"h", app=None, proc=None, msgid=None, msg=None, full=None, sd=None, fac=None, sev=None, ts=1.5):
    return {"ts_bits": f64(ts), "fac": fac, "sev": sev, "host": host, "app": app, "proc": proc, "msgid": msgid, "msg": msg,
            "full": full, "sd": sd}


class _Watched(O._Message):
    """the oracle's message, with every allocation and the pointer that reaches it logged"""

    def __init__(self):
        super().__init__()
        self.log = []

    def point(self, ps, pw, place, kind, hi):
        super().point(ps, pw, place, kind, hi)
        self.log.append((ps, pw, place, kind, hi))


def check_layout(emu, rec, extra=()):
    m = _Watched()
    msg = O.encode(rec, list(extra), m)
    n = len(m.log)
    typ, val, cont, off = (np.zeros(n, np.int32), np.zeros(n, np.uint32), np.zeros(n, np.int32), np.zeros(n, np.uint32))
    words = []
    for t, (ps, pw, (s, pos, pad), kind, hi) in enumerate(m.log):
        if kind == 0:
            typ[t], nw = 0, 11
        elif hi & 7 == 2:
            typ[t], val[t] = 1, (hi >> 3) - 1
            nw = (val[t] + 8) // 8
        else:
            typ[t], val[t] = 2, (hi >> 3) // 4
            nw = 1 + 4 * val[t]
        words.append(nw)
        holders = [u for u in range(t) if m.log[u][2][0] == ps and m.log[u][2][1] <= pw < m.log[u][2][1] + words[u]]
        cont[t] = holders[-1] if holders else -1
        off[t] = pw - m.log[cont[t]][2][1] if holders else pw
    seg, pad = np.zeros(n, np.int32), np.zeros(n, np.int32)
    pos = np.zeros(n, np.uint32)
    ptr, padw = np.zeros(n, np.uint64), np.zeros(n, np.uint64)
    table, ntable, nbytes = np.zeros(40, np.uint64), C.c_int32(), C.c_ulonglong()
    rc = emu.emu_capnp_layout(n, typ.ctypes.data, val.ctypes.data, cont.ctypes.data, off.ctypes.data, seg.ctypes.data,
                              pos.ctypes.data, pad.ctypes.data, ptr.ctypes.data, padw.ctypes.data, table.ctypes.data,
                              C.byref(ntable), C.byref(nbytes))
    assert rc == 0
    for t, (ps, pw, (s, p, pd), kind, hi) in enumerate(m.log):
        assert (seg[t], pos[t], pad[t]) == (s, p, -1 if pd is None else pd), t
        assert int(ptr[t]) == m.words[ps][pw], t
        if pd is not None:
            assert int(padw[t]) == m.words[s][pd], t
    assert nbytes.value == len(msg)
    assert table[:ntable.value].tobytes() == msg[:8 * ntable.value]
    got, got_extra = O.read(msg)
    assert got == O.as_read(rec) and got_extra == list(extra)
    return msg, len(m.size)


def test_reference_tests_and_pair_tag(emu):
    doc = json.loads((HERE / "golden" / "capnp_encoder_tests.json").read_text())
    for case in doc["cases"]:
        r = case["record"]
        sd = None
        if r["sd"] is not None:
            sd = []
            for e in r["sd"]:
                pairs = []
                for k, v in e["pairs"]:
                    (member, value), = v.items()
                    pairs.append((k.encode(), (member, value.encode() if member == "string" else f64(value))))
                sd.append((e["sd_id"].encode() if e["sd_id"] else None, pairs))
        rec = record(host=r["hostname"].encode(), app=r["appname"].encode(), proc=r["procid"].encode(), msg=r["msg"].encode(),
                     full=r["full_msg"].encode(), sd=sd, fac=r["facility"], sev=r["severity"], ts=r["ts"])
        msg, _ = check_layout(emu, rec, [(k.encode(), v.encode()) for k, v in case["extra"]])
        assert msg.decode("utf-8", "replace") == case["lossy"], case["source"]
    for n in (0, 1, 2, 1000, (1 << 27) - 1):
        assert emu.emu_capnp_pairs_tag(n) == (n << 2) | ((2 | (2 << 16)) << 32)


@pytest.mark.parametrize("n", [0, 1, 6, 7, 8, 9, 15, 16, 17])
def test_text_lengths(emu, n):
    text = bytes(97 + j % 26 for j in range(n))
    msg, _ = check_layout(emu, record(host=text, msg=text, sd=[(text, [(b"_" + text, ("string", text))])]), [(text, text)])
    assert len(msg) % 8 == 0


@pytest.mark.parametrize("words", range(1020, 1029))
def test_segment_zero_edge(emu, words):
    """a message of 1020..1028 words: root pointer + Record + host (1 word) + msg; one segment up to 1024"""
    msg_words = words - 1 - 11 - 1
    rec = record(host=b"", msg=b"m" * (8 * msg_words - 1))
    msg, nseg = check_layout(emu, rec)
    assert nseg == (1 if words <= 1024 else 2)


def test_backfill_and_straddling_extras(emu):
    # a message too large for segment 0 goes to segment 1; the smaller objects after it still fill segment 0
    rec = record(msg=b"M" * 9000, full=b"f" * 40, sd=[(b"id", [(b"_k", ("string", b"v" * 30))] * 3)])
    _, nseg = check_layout(emu, rec, [(b"a", b"1"), (b"b", b"2")])
    assert nseg == 2
    # extras whose list or texts meet the end of segment 0, at every word around it
    for pad in range(0, 120, 3):
        rec = record(msg=b"m" * (8 * (1024 - 12 - 1 - 6 - 18) - 1 + pad))
        check_layout(emu, rec, [(b"x-header1", b"header1 value"), (b"y", b""), (b"z" * 20, b"w" * 20)])


@pytest.mark.parametrize("n", [0, 1, 1000])
def test_pair_counts(emu, n):
    pairs = [(b"_k%d" % j, ("string", b"v" * (j % 17))) for j in range(n)]
    check_layout(emu, record(app=b"a", proc=b"p", msgid=b"m", msg=b"x", full=b"y", sd=[(b"id@1", pairs)], fac=3, sev=4))
    check_layout(emu, record(sd=[(None, pairs)]) if n else record(sd=[(b"id", [])]))


def test_every_member(emu):
    pairs = [(b"_s", ("string", b"str")), (b"_t", ("bool", True)), (b"_f", ("bool", False)), (b"_d", ("f64", f64(-0.0))),
             (b"_n", ("f64", 0x7FF8000000000001)), (b"_i", ("i64", -(1 << 63))), (b"_u", ("u64", (1 << 64) - 1)),
             (b"_z", ("null", None)), (b"_e", ("string", b""))]
    msg, _ = check_layout(emu, record(sd=[(None, pairs)], fac=0, sev=7))
    assert O.read(msg)[0]["sd"][0][1] == pairs


def test_random_multi_segment(emu):
    rng = random.Random(7)
    for _ in range(300):
        def txt():
            return b"t" * rng.choice([0, 1, 7, 8, 100, 3000, 9000, 20000, 70000])
        pairs = [(b"_" + txt(), ("string", txt()) if rng.random() < 0.7 else ("u64", rng.getrandbits(64)))
                 for _ in range(rng.choice([0, 1, 3, 40]))]
        rec = record(host=txt(), app=txt() if rng.random() < 0.5 else None, msg=txt(), full=txt(),
                     sd=[(txt() if rng.random() < 0.5 else None, pairs)] if pairs or rng.random() < 0.3 else None)
        check_layout(emu, rec, [(b"x%d" % j, txt()) for j in range(rng.choice([0, 0, 2, 5]))])


# ---- the segment list model of tests/capnp_out_edges.py ---------------------------------------------------------------

def test_segment_model_random_records():
    """the model's entries, joined, are the oracle's message for the 300 random multi-segment records"""
    rng = random.Random(7)
    for _ in range(300):
        def txt():
            return b"t" * rng.choice([0, 1, 7, 8, 100, 3000, 9000, 20000, 70000])
        pairs = [(b"_" + txt(), ("string", txt()) if rng.random() < 0.7 else ("u64", rng.getrandbits(64)))
                 for _ in range(rng.choice([0, 1, 3, 40]))]
        rec = record(host=txt(), app=txt() if rng.random() < 0.5 else None, msg=txt(), full=txt(),
                     sd=[(txt() if rng.random() < 0.5 else None, pairs)] if pairs or rng.random() < 0.3 else None)
        extra = [(b"x%d" % j, txt()) for j in range(rng.choice([0, 0, 2, 5]))]
        assert b"".join(b for _, b in CE.segments(rec, extra)) == O.encode(rec, extra)


@pytest.mark.parametrize("src", [CE.R5, CE.LTSV, CE.GELF, CE.R3])
def test_window_lines_model(oracle, src):
    """every window line's record: the model joins to the oracle's message, and the lines reach every (boundary, kind)
    cell, every total and every after-a-list cell they claim, with and without extras"""
    lines = CE.window_lines(src)
    cfg = oracle.LtsvConfig(CE.TYPED, CE.SUFFIXES) if src == CE.LTSV else oracle.Rfc3164Config(2026) if src == CE.R3 else None
    recs = O.decode_records(oracle, src, *oracle.pack(lines), cfg=cfg)
    assert all(r is not None for r in recs)
    cells, totals, after = set(), set(), set()
    for extra in ([], O.extra_pairs(CE.EXTRA)):
        for r in recs:
            assert b"".join(b for _, b in CE.segments(r, extra, src)) == O.encode(r, extra)
            c, t, a = CE.cells(r, extra, src)
            cells, after = cells | c, after | a
            totals.add(t)
    assert not {(b, k) for b in CE.BOUNDARIES for k in CE.KINDS[src]} - cells
    assert not CE.AFTER_LIST[src] - after
    if src != CE.R3:
        assert set(CE.TOTALS) <= totals
    if src != CE.R3:  # lane_lines' records end on the window boundaries or take four windows
        shapes = CE.LANE_SHAPES[src]
        got = [len(CE.segments(r, [], src)) for r in O.decode_records(
            oracle, src, *oracle.pack([CE.lane_line(src, *shapes[k]) for k in (64, 128, 4)]), cfg=cfg)]
        assert got[:2] == [64, 128] and 192 < got[2] <= 256
