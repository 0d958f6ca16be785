"""Side-table regrow on every entry point that redoes a batch after a bump table overflowed: the first call on a fresh
context must overflow, grow the table to the reported need, redo the batch and still match the oracle.  A second call
on the same context fits at once, so the first call's kernel launches are a multiple of the second's.  GPU only."""
import numpy as np
import pytest

import vectors as V

pytestmark = pytest.mark.gpu
R5, LTSV, GELF = 0, 1, 2

# 400 one-pair elements per line: the rows go to the RFC5424 8-byte entries and wide tables, far past their first sizes
R5_LINES = [(V.H + "".join('[i k="v"]' for _ in range(400)) + " m").encode()] * 900
# 1 MiB contexts start with max(1 MiB / 24, 4096) = 43 Ki side-table rows; 1000 lines of 100 members need 100 k
GELF_LINES = [(b'{"version":"1.1","host":"h","short_message":"m","timestamp":1,'
               + b",".join(b'"_k%02d":%d' % (k, i % 10) for k in range(100)) + b"}") for i in range(1000)]
LTSV_LINES = [b"time:[2015-08-05T15:53:45Z]\thost:h\tmessage:m" + b"".join(b"\tk%02d:%d" % (k, i % 10) for k in range(100))
              for i in range(1000)]


def _decode(dec, oracle, fmt, lines):
    data, offs = oracle.pack(lines)
    res = dec.decode(data, offs)
    return dec.dump(res, data, offs), oracle.decode_dump(fmt, data, offs)


def _resident(dec, oracle, fmt, lines):
    data, offs = oracle.pack(lines)
    dec.upload(data, offs)
    dec.parse_resident()
    res = dec.download()
    return dec.dump(res, data, offs), oracle.decode_dump(fmt, data, offs)


def _split(dec, oracle, fmt, lines):
    stream = np.frombuffer(b"\n".join(lines) + b"\n", dtype=np.uint8).copy()
    buf, bo, _, _ = dec.split_dump(stream)
    data, offs = oracle.pack(lines)
    return (buf, bo), oracle.decode_dump(fmt, data, offs)


def _encode(dec, oracle, fmt, lines):
    data, offs = oracle.pack(lines)
    buf, o, _, _ = dec.decode_encode_gelf(data, offs)
    return (buf, o), oracle.decode_encode_gelf(fmt, data, offs, {}, nthreads=16)


@pytest.mark.parametrize("entry,fmt,lines,max_bytes", [
    ("split", R5, R5_LINES, 8 << 20),
    ("resident", R5, R5_LINES, 8 << 20),
    ("decode", GELF, GELF_LINES, 1 << 20),
    ("decode", LTSV, LTSV_LINES, 1 << 20),
    ("encode", R5, R5_LINES, 8 << 20),
], ids=["split-rfc5424", "resident-rfc5424", "decode-gelf", "decode-ltsv", "encode-rfc5424"])
def test_side_table_regrow(native, oracle, entry, fmt, lines, max_bytes):
    run = {"split": _split, "resident": _resident, "decode": _decode, "encode": _encode}[entry]
    dec = native.BatchDecoder(fmt, max_batch_bytes=max_bytes, max_batch_lines=len(lines))
    try:
        launches = []
        for _ in range(2):
            n0 = dec.kernel_launches()
            (gbuf, goffs), (obuf, ooffs) = run(dec, oracle, fmt, lines)
            launches.append(dec.kernel_launches() - n0)
            assert gbuf == obuf and np.array_equal(goffs, ooffs)
        assert launches[0] == 2 * launches[1], launches  # the first call overflowed and redid the batch once
    finally:
        dec.close()
