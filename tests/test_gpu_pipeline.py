"""Config #1 plumbing (stdin + line framing + RFC5424, SURVEY.md §3.2) through the batching splitter, and the
multi-context fan-out. GPU only."""
import numpy as np
import pytest

import vectors as V

pytestmark = pytest.mark.gpu


def test_config1_stdin_10k_lines(native, oracle):
    """10 000-line RFC5424 'file': BatchingLineSplitter (GPU decode) must emit exactly what LineSplitter +
    the reference decoder would: same records in order, same stderr text for bad lines (line_splitter.rs:37-39)."""
    data, offs = native.generate(native.FMT_RFC5424, 1, 10_000, bad_frac=0.01)
    lines = [bytes(data[offs[i]:offs[i + 1]]) for i in range(10_000)]
    lines[17] = lines[17] + b"\r"            # CRLF line: BufRead::lines strips the '\r'
    lines[4000] = b"<13>1 \xff\xfe broken utf8"  # InvalidData -> "Invalid UTF-8 input", skipped
    lines[5000] = b""                         # empty line -> "Unsupported BOM: []"
    text = b"\n".join(lines) + b"\n"
    dec = native.BatchDecoder(native.FMT_RFC5424, max_batch_bytes=64 << 20, max_batch_lines=1 << 16)
    try:
        records, err, out = native.splitter_run(dec, text, max_lines=3000, max_bytes=1 << 20)
    finally:
        dec.close()
    # expected, from the oracle applied line by line to what LineSplitter would hand to decode()
    fed = [l[:-1] if (i == 17) else l for i, l in enumerate(lines) if i != 4000]
    d, o = oracle.pack(fed)
    buf, bo = oracle.decode_dump(0, d, o)
    exp_records, exp_err = [], []
    k = 0
    for i, l in enumerate(lines):
        if i == 4000:
            exp_err.append(b"Invalid UTF-8 input")
            continue
        dump = buf[bo[k]:bo[k + 1]]
        line = fed[k]
        k += 1
        if dump.startswith(b"E:"):
            msg = dump[2:dump.index(b";out=")]
            exp_err.append(msg + b": [" + line.decode().strip().encode() + b"]")
        else:
            exp_records.append(dump[:dump.rindex(b";out=")] + b";out=0")
    assert records.split(b"\n")[:-1] == exp_records
    assert err.split(b"\n")[:-1] == exp_err
    assert out == b""


def test_single_line_decoder_trait(native, oracle):
    """Decoder::decode(line) drop-in: a batch of one through the same kernels."""
    dec = native.BatchDecoder(native.FMT_RFC5424)
    try:
        for line in (V.G1_LINE, V.G2_LINE, "abc", ""):
            data, offs = oracle.pack([line.encode()])
            res = dec.decode(data, offs)
            g, _ = dec.dump(res, data, offs, nthreads=1)
            r, _ = oracle.decode_dump(0, data, offs, nthreads=1)
            assert g == r
    finally:
        dec.close()


def test_multi_context_fanout(native, oracle):
    """MultiGpuBatchDecoder host logic (sharding, per-context threads, ordered gather) with two contexts on GPU 0;
    the same on two REAL devices is tests/test_gpu_fullsize.py::test_multi_device_fanout (two GPUs)."""
    devices = [0, 0]
    data, offs = native.generate(native.FMT_RFC5424, 77, 400_000)
    gbuf, goffs = native.multi_gpu_decode_dump(native.FMT_RFC5424, devices, data, offs)
    obuf, ooffs = oracle.decode_dump(0, data, offs)
    assert gbuf == obuf and np.array_equal(goffs, ooffs)
    # fewer lines than shards
    d2, o2 = oracle.pack([V.G1_LINE.encode()])
    gbuf, _ = native.multi_gpu_decode_dump(native.FMT_RFC5424, devices + devices, d2, o2)
    obuf, _ = oracle.decode_dump(0, d2, o2)
    assert gbuf == obuf


def test_capacity_and_argument_errors(native, oracle):
    dec = native.BatchDecoder(native.FMT_RFC5424, max_batch_bytes=8 << 20, max_batch_lines=1000)
    try:
        data, offs = native.generate(native.FMT_RFC5424, 3, 5000)
        with pytest.raises(RuntimeError, match="max_batch_lines|more lines"):
            dec.decode(data, offs)
        bad2 = np.array([10, 5], dtype=np.int32)
        with pytest.raises(RuntimeError, match="non-decreasing"):
            dec.decode(data, bad2)
        # a non-monotone offset INSIDE the batch is caught by the device-side check next to the parse: FG_E_ARG, no kernel
        # ever sees the bad extent, and the context stays usable
        bad = offs[:10].copy()
        bad[5] = bad[9] + 5
        with pytest.raises(RuntimeError, match="non-decreasing"):
            dec.decode(data, bad)
        good = offs[:10].copy()
        assert dec.decode(data, good).n == 9
        # structured-data table overflow triggers a regrow, not a failure
        lines = [(V.H + "".join('[i k="v"]' for _ in range(400)) + " m").encode()] * 900
        d2, o2 = oracle.pack(lines)
        res = dec.decode(d2, o2)
        # 400 one-pair elements per line: 16 bytes of side-table rows per 9 input bytes do not fit behind the cursor, so these
        # lines take the slow path and their rows land in the wide table — which regrows from 4 Ki rows
        assert int(res.raw.n_entries8) + int(res.n_entries) == 900 * 800 and int(res.raw.n_wide) == 900
        g, _ = dec.dump(res, d2, o2)
        r, _ = oracle.decode_dump(0, d2, o2)
        assert g == r
    finally:
        dec.close()


def test_splitter_line_larger_than_a_batch(native, oracle):
    """ADVICE r1: a single line longer than the decoder's max_batch_bytes must not abort the stream — the reference's
    LineSplitter takes lines of any length.  It is decoded on a context of its own; order of records is kept."""
    big = b"<13>1 " + V.TS.encode() + b" h a p m - " + b"y" * (3 << 20)
    lines = [V.G1_LINE.encode(), big, V.G2_LINE.encode(), b"abc"]
    text = b"\n".join(lines) + b"\n"
    dec = native.BatchDecoder(native.FMT_RFC5424, max_batch_bytes=1 << 20, max_batch_lines=1024)
    try:
        records, err, out = native.splitter_run(dec, text, max_lines=1 << 16, max_bytes=64 << 20)
    finally:
        dec.close()
    d, o = oracle.pack(lines)
    buf, bo = oracle.decode_dump(0, d, o)
    dumps = [buf[bo[i]:bo[i + 1]] for i in range(4)]
    assert records.split(b"\n")[:-1] == [x[:x.rindex(b";out=")] + b";out=0" for x in dumps[:3]]
    assert err == b"Unsupported BOM: [abc]\n"


def _expected(oracle, lines, quiet_blank=False):
    d, o = oracle.pack(lines)
    buf, bo = oracle.decode_dump(0, d, o)
    recs, errs = [], []
    for i, l in enumerate(lines):
        dump = buf[bo[i]:bo[i + 1]]
        if dump.startswith(b"E:"):
            t = l.decode().strip().encode()
            if not (quiet_blank and not t):
                errs.append(dump[2:dump.index(b";out=")] + b": [" + t + b"]")
        else:
            recs.append(dump[:dump.rindex(b";out=")] + b";out=0")
    return recs, errs


def test_nul_and_syslen_batching_splitters(native, oracle):
    """Batching twins of NulSplitter (nul_splitter.rs:10-47: NUL-terminated records, no message for a blank rejected
    record) and SyslenSplitter (syslen_splitter.rs:10-57: "<len> <record>", stream ends with "Can't read message's
    length")."""
    data, offs = native.generate(native.FMT_RFC5424, 5, 3000, bad_frac=0.02)
    lines = [bytes(data[offs[i]:offs[i + 1]]) for i in range(3000)]
    lines[10] = b""            # blank record: rejected ("Unsupported BOM") but not reported by the NUL splitter
    lines[11] = b"   "
    lines[12] = lines[12] + b"\r\n"  # '\r' / '\n' are ordinary bytes under NUL and syslen framing
    dec = native.BatchDecoder(native.FMT_RFC5424, max_batch_bytes=8 << 20, max_batch_lines=1 << 12)
    try:
        recs, errs = _expected(oracle, lines, quiet_blank=True)
        records, err, _ = native.splitter_run(dec, b"\0".join(lines) + b"\0", max_lines=700, framing=1)
        assert records.split(b"\n")[:-1] == recs and err.split(b"\n")[:-1] == errs
        # syslen: the newline inside record 12 must survive (records are split on b";out=0\n" here)
        recs, errs = _expected(oracle, lines)
        text = b"".join(b"%d %s" % (len(l), l) for l in lines)
        records, err, _ = native.splitter_run(dec, text + b"12 short", max_lines=700, framing=2)
        assert records.split(b"\n")[:-1] == recs
        assert err.split(b"\n")[:-1] == errs + [b"failed to fill whole buffer"]
        records, err, _ = native.splitter_run(dec, text + b"x1 abc", max_lines=700, framing=2)
        assert err.split(b"\n")[:-1] == errs + [b"Can't read message's length"]
    finally:
        dec.close()
