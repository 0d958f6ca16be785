"""The passthrough oracle (tests/passthrough_oracle.py) against the reference's own encoder tests
(tests/golden/passthrough_encoder_tests.json, passthrough_encoder.rs:52-143), and its Record.full_msg per input format
against the decoders' rules.  No GPU needed."""
import json
from pathlib import Path

import numpy as np

import passthrough_oracle as O

GOLDEN_DIR = Path(__file__).resolve().parent / "golden"
GOLDEN = json.loads((GOLDEN_DIR / "passthrough_encoder_tests.json").read_text())


def test_reference_encoder_tests():
    assert len(GOLDEN["cases"]) + len(GOLDEN["not_applicable"]) == 4
    for case in GOLDEN["cases"]:
        full = case["record"]["full_msg"]
        header = (case["header"] or "").encode()
        got = O.encode(None if full is None else full.encode(), header)
        if case["error"] is None:
            assert got == case["expected"].encode(), case["source"]
        else:
            assert got is None and case["error"] == O.NO_RAW, case["source"]


def _pack(lines):
    offs = np.zeros(len(lines) + 1, np.int32)
    np.cumsum([len(l) for l in lines], out=offs[1:])
    data = np.frombuffer(b"".join(lines), np.uint8).copy()
    return data, offs


def test_full_msg_per_input_format(oracle):
    """full_msg as each decoder gives it: RFC5424 after the BOM and trim_end, RFC3164 the trimmed line, LTSV untrimmed,
    GELF the unescaped full_message (None when absent)"""
    r5 = b"<13>1 2015-08-05T15:53:45Z h a p m - \xef\xbb\xbfmsg \t\xc2\xa0\xe3\x80\x80"
    d, o = _pack([r5])
    recs, no_raw = O.decode_encode_passthrough(oracle, 0, d, o, header=b"H")
    assert recs == [b"H<13>1 2015-08-05T15:53:45Z h a p m - \xef\xbb\xbfmsg"] and no_raw == [False]
    d, o = _pack([b"host:h\ttime:1\tmessage:m  "])
    assert O.decode_encode_passthrough(oracle, 1, d, o)[0] == [b"host:h\ttime:1\tmessage:m  "]
    d, o = _pack([b'{"host":"h","short_message":"m","full_message":"a\\tb\\u00e9"}', b'{"host":"h","short_message":"m"}',
                  b'{"host":"h","short_message":"m","full_message":""}'])
    recs, no_raw = O.decode_encode_passthrough(oracle, 2, d, o, header=b"<")
    assert recs == [b"<a\tb\xc3\xa9", b"", b"<"] and no_raw == [False, True, False]


def test_encoder_status_text(native):
    """FG_EP_NO_RAW lies above every decoder and framing status, and its text is the reference encoder's literal
    (tests/golden/encoder_strings.json), as the oracle has it"""
    assert O.FG_EP_NO_RAW >= native.load_cuda().fg_error_count()
    literals = [s for per_file in json.loads((GOLDEN_DIR / "encoder_strings.json").read_text())["literals"].values() for s in per_file]
    for fmt in range(4):
        assert native.error_string(fmt, O.FG_EP_NO_RAW) == O.NO_RAW
    assert O.NO_RAW in literals
    assert native.error_string(0, O.FG_EP_NO_RAW + 1) is None
