"""The kernels at their capacity limits on the device: the batches of kernel_edges.py through the C ABI against the
oracle (fg_decode_batch, the resident path, fg_split_decode, the fused GELF encoder).  RFC5424 makes the tile choice
observable: FG_FLAG_WIDE must be set on exactly the lines the restated pick_tile says do not fit.  GPU only."""
import ctypes
import os

import numpy as np
import pytest

import kernel_edges as K
from conftest import assert_parity

pytestmark = pytest.mark.gpu
YEAR = 2026
FLAG_WIDE = 0x80


def smem_optin() -> int:
    rt = ctypes.CDLL("libcudart.so")
    v = ctypes.c_int(0)
    assert rt.cudaDeviceGetAttribute(ctypes.byref(v), 97, 0) == 0  # cudaDevAttrMaxSharedMemoryPerBlockOptin
    return v.value


@pytest.fixture(scope="module")
def decs(native):
    out = {}

    def get(fmt, **kw):
        key = (fmt, repr(sorted(kw.items())))
        if key not in out:
            out[key] = native.BatchDecoder(fmt, max_batch_bytes=64 << 20, max_batch_lines=1 << 20,
                                           rfc3164_year=YEAR if fmt == K.R3164 else 0, **kw)
        return out[key]
    yield get
    for d in out.values():
        d.close()


def cfg_of(oracle, fmt, schema=None, suffixes=None):
    if fmt == K.R3164:
        return oracle.Rfc3164Config(YEAR)
    if fmt == K.LTSV and schema is not None:
        return oracle.LtsvConfig(schema, suffixes)
    return None


def wide_set(res) -> set[int]:
    return set(np.flatnonzero((res.meta >> 24) & FLAG_WIDE).tolist())


def test_r5_rounds_at_the_maximum_tile(decs, oracle):
    """A batch whose mean clamps pick_tile at this device's RFC5424 maximum (derived from its opt-in shared memory per
    block): the parse kernel runs with its largest tile, CTA spans beyond it are cut into rounds, and only the lines over
    65535 bytes go wide.  The other RFC5424 batches here use tiles up to 66560, which must stay below the maximum."""
    optin = smem_optin()
    max5 = K.max_tile5(optin)
    print(f"sharedMemPerBlockOptin = {optin}, RFC5424 max tile = {max5}")
    assert max5 > K.R5_TILE_16BIT
    lines = K.r5_max_tile(seed=310)
    data, offs = K.pack(lines)
    assert K.pick_tile(K.R5, int(offs[-1]), len(lines), max5=max5) == max5 and int(offs[64] - offs[0]) > max5
    dec = decs(K.R5)
    for resident in (False, True):
        res = assert_parity(dec, oracle, K.R5, data, offs, resident=resident)
        assert wide_set(res) == K.r5_long_wide(lines) and len(wide_set(res)) == 4


@pytest.mark.parametrize("fmt", [K.R5, K.LTSV, K.GELF, K.R3164])
def test_tile_fit_every_alignment(decs, oracle, fmt):
    for tile in ((8192, 20480) if fmt == K.R5 else (8192,)):
        data, offs, info = K.tile_fit(fmt, tile, seed=100 + fmt + tile)
        assert K.batch_tile(fmt, offs) == tile
        dec = decs(fmt)
        for resident in (False, True):
            res = assert_parity(dec, oracle, fmt, data, offs, cfg_of(oracle, fmt), resident=resident)
            if fmt == K.R5:
                assert wide_set(res) == set(info["over"]), f"tile {tile}"
        print(f"fmt {fmt}: tile {tile}, lines {len(offs) - 1}, over the tile {len(info['over'])}")


@pytest.mark.parametrize("fmt", [K.R5, K.LTSV, K.GELF])
def test_stale_odd_granule(decs, oracle, fmt):
    data, offs, tile = K.stale_granule(fmt, seed=200 + fmt)
    assert K.stale_rounds(offs, tile) == 32
    assert_parity(decs(fmt), oracle, fmt, data, offs)


def test_r5_sixteen_bit_lines(decs, oracle):
    lines, tile = K.r5_sixteen_bit(seed=300)
    want = K.r5_long_wide(lines)
    data, offs = K.pack(lines)
    assert K.batch_tile(K.R5, offs) == tile
    dec = decs(K.R5)
    res = assert_parity(dec, oracle, K.R5, data, offs)
    assert wide_set(res) == want and len(want) == 4
    # device framing: the same lines with "\n" and "\r\n" (the 16-bit test is on the stripped length)
    d0, o0 = K.pack(lines)
    obuf, ooffs = oracle.decode_dump(K.R5, d0, o0, None, nthreads=os.cpu_count() or 4)
    for crlf in (False, True):
        stream = np.frombuffer(K.with_terminators(lines, crlf), dtype=np.uint8)
        assert K.pick_tile(K.R5, len(stream), len(lines)) >= 65536 + 32
        buf, bo, line_offs, _ = dec.split_dump(stream)
        assert len(bo) == len(lines) + 1
        assert [buf[bo[i]:bo[i + 1]] for i in range(len(lines))] == [obuf[ooffs[i]:ooffs[i + 1]] for i in range(len(lines))]
        assert wide_set(dec.split_decode(stream)) == want


def test_ltsv_slots_direct_next_and_sixteen_bit(decs, oracle):
    dec = decs(K.LTSV)
    data, offs, info = K.ltsv_slots(seed=400)
    assert K.batch_tile(K.LTSV, offs) == info["tile"]
    assert_parity(dec, oracle, K.LTSV, data, offs)
    assert_parity(dec, oracle, K.LTSV, data, offs, resident=True)
    data, offs, tile = K.ltsv_sixteen_bit(seed=500)
    assert K.batch_tile(K.LTSV, offs) == tile
    assert_parity(dec, oracle, K.LTSV, data, offs)


@pytest.mark.parametrize("label", [s[0] for s in K.ltsv_schemas()])
def test_ltsv_schema_placement(decs, oracle, label):
    _, schema, suffixes = next(s for s in K.ltsv_schemas() if s[0] == label)
    data, offs = K.pack(K.ltsv_schema_lines(schema, suffixes, seed=600))
    dec = decs(K.LTSV, ltsv_schema=schema, ltsv_suffixes=suffixes)
    assert_parity(dec, oracle, K.LTSV, data, offs, cfg_of(oracle, K.LTSV, schema, suffixes))


def test_gelf_slots_members_and_numbers(decs, oracle):
    data, offs, info = K.gelf_slots(seed=700)
    assert K.batch_tile(K.GELF, offs) == info["tile"]
    assert_parity(decs(K.GELF), oracle, K.GELF, data, offs)
    assert_parity(decs(K.GELF), oracle, K.GELF, data, offs, resident=True)


@pytest.mark.parametrize("fmt", [K.LTSV, K.GELF, K.R3164])
def test_one_odd_line_at_every_lane(decs, oracle, fmt):
    data, offs = K.lane_mix(fmt, seed=800 + fmt)
    assert_parity(decs(fmt), oracle, fmt, data, offs, cfg_of(oracle, fmt))


# ---- the fused GELF encoder -------------------------------------------------------------------------------------------

def enc_check(dec, oracle, lines, extra=None):
    data, offs = K.pack(lines)
    dec.set_gelf_extra(extra or {})
    buf, o, status, _ = dec.decode_encode_gelf(data, offs)
    obuf, oo = oracle.decode_encode_gelf(K.R5, data, offs, extra or {}, nthreads=os.cpu_count() or 4)
    if buf != obuf or not np.array_equal(o, oo):
        for i in range(len(lines)):
            a, b = buf[o[i]:o[i + 1]], obuf[oo[i]:oo[i + 1]]
            assert a == b, (i, lines[i][:300], a[:400], b[:400])
        raise AssertionError("record offsets differ")
    return status


def test_encoder_segment_windows_and_pair_modes(decs, oracle):
    """0..40 pairs (segment totals across 56 and 112), empty values and hosts; duplicates around the 24-pair switch to
    the O(n^2) selection, where the last duplicate must win as it does in the local mode."""
    dec = decs(K.R5)
    enc_check(dec, oracle, K.enc_pair_counts(seed=900))
    enc_check(dec, oracle, K.enc_duplicates(seed=901))


@pytest.mark.parametrize("k", range(len(K.ENC_EXTRAS)))
def test_encoder_extras_against_sd_names(decs, oracle, k):
    """output.gelf_extra keys that sort before '_', equal '_', collide with an SD name, hold a byte >= 0x80, are empty."""
    dec = decs(K.R5)
    enc_check(dec, oracle, K.enc_pair_counts(seed=902)[::3] + K.enc_duplicates(seed=903), K.ENC_EXTRAS[k])


def test_encoder_long_records_spans_and_lanes(decs, oracle):
    """records of >= 1008 bytes (length class 63); a 256-line span larger than the encoder tile; warps with a rejected
    line and a line of more than 24 pairs at every lane position."""
    dec = decs(K.R5)
    long_lines, span = K.enc_long_and_spans(seed=904)
    enc_check(dec, oracle, long_lines)
    d, o = K.pack(span)
    tile = K.batch_tile(K.R5, o)
    assert int(o[256 * 5] - o[256 * 4]) > min(4 * tile, K.H100_MAX_TILE5)
    enc_check(dec, oracle, span)
    status = enc_check(dec, oracle, K.enc_lane_mix(seed=905))
    assert int((status != 0).sum()) == 32


# ---- UTF-8 and framing seams of the device splitter ---------------------------------------------------------------------

@pytest.mark.parametrize("framing", [0, 1])
def test_split_utf8_and_framing_seams(decs, oracle, framing):
    import pysplit
    stream = K.utf8_stream(b"\0" if framing else b"\n", seed=906)
    offs, lines, valid = (pysplit.split_nul if framing else pysplit.split_lines)(stream)
    assert 0 < sum(valid) < len(valid)
    buf, bo, line_offs, _ = decs(K.R5).split_dump(np.frombuffer(stream, dtype=np.uint8), framing)
    assert np.array_equal(line_offs, offs)
    good = [l for l, v in zip(lines, valid) if v]
    d, o = K.pack(good)
    obuf, oo = oracle.decode_dump(K.R5, d, o, nthreads=os.cpu_count() or 4)
    k = 0
    for i, (l, v) in enumerate(zip(lines, valid)):
        got = buf[bo[i]:bo[i + 1]]
        if not v:
            assert got == b"E:Invalid UTF-8 input;out=0", (i, l[-40:], got)
        else:
            assert got == obuf[oo[k]:oo[k + 1]], (i, l[-40:], got)
            k += 1
