"""CPU check of the kernels at their capacity limits: the batches of kernel_edges.py run through the emulation of the
device logic (tests/emu) with the tile the host would pick, are compared with the oracle, and the emulation's path
counters must show that every targeted path was taken — as an exact count where kernel_edges restates the round logic.
No GPU needed; test_gpu_kernel_edges.py sends the same batches through the C ABI."""
import numpy as np
import pytest

import kernel_edges as K
from conftest import first_diff

YEAR = 2026


@pytest.fixture(scope="module")
def emu():
    import sys
    from pathlib import Path
    sys.path.insert(0, str(Path(__file__).resolve().parent / "emu"))
    import emu as E
    E.build()
    return E


def same(got, want, data, offs):
    gbuf, goffs = got
    obuf, ooffs = want
    if not (gbuf == obuf and np.array_equal(goffs, ooffs)):
        diffs = first_diff(gbuf, goffs, obuf, ooffs, data, offs)
        msg = "\n".join(f"line {i}: {line[:200]!r}\n   emu: {g[:300]!r}\n   ref: {o[:300]!r}" for i, line, g, o in diffs)
        raise AssertionError(f"{len(diffs)}+ lines differ from the oracle:\n{msg}")


def run(emu, native, oracle, fmt, data, offs, tile, cfg=None, **kw):
    """emulated decode at `tile` == oracle; returns the emulation's path counters"""
    if fmt == K.R5:
        buf, o, info = emu.decode_dump(native, data, offs, tile_bytes=tile, **kw)
    elif fmt == K.LTSV:
        buf, o, info = emu.ltsv_decode_dump(native, data, offs, tile_bytes=tile, **kw)
    elif fmt == K.GELF:
        buf, o, info = emu.gelf_decode_dump(native, data, offs, tile_bytes=tile, **kw)
    else:
        buf, o, info = emu.r3164_decode_dump(native, data, offs, YEAR, tile_bytes=tile, **kw)
        cfg = oracle.Rfc3164Config(YEAR)
    same((buf, o), oracle.decode_dump(fmt, data, offs, cfg, nthreads=8), data, offs)
    return info


def repeated_time(lines):
    return {i for i, l in enumerate(lines) if sum(p.startswith(b"time:") for p in l.split(b"\t")) > 1}


@pytest.mark.parametrize("fmt", [K.R5, K.LTSV, K.GELF, K.R3164])
def test_tile_fit_every_alignment(emu, native, oracle, fmt):
    """Lines whose aligned span is tile - 1, tile, tile + 1 at every start offset mod 16, first in a CTA and after a
    cut round, and CTAs of >= 3 TMA rounds around r == 0 lines: exactly the lines over the tile leave it."""
    for tile in ((8192, 20480) if fmt == K.R5 else (8192,)):
        data, offs, info = K.tile_fit(fmt, tile, seed=100 + fmt + tile)
        assert K.batch_tile(fmt, offs) == tile and len(info["over"]) == 16 * 2 + 6
        c = run(emu, native, oracle, fmt, data, offs, tile)
        lines = K.lines_of(data, offs)
        if fmt == K.R5:
            assert c["wide_lines"] == set(info["over"])  # every line is regular: only the tile sends a line wide
        elif fmt == K.R3164:
            assert (c["from_tile"], c["from_global"]) == K.r3164_tile_split(offs, tile)
            assert c["from_global"] >= len(info["over"])
        else:
            parts = K.ltsv_parts(lines) if fmt == K.LTSV else K.gelf_members(lines)
            want = K.slot_rounds(offs, tile, parts, K.LTSV_SLOTS if fmt == K.LTSV else K.GELF_SLOTS, fmt == K.LTSV)
            assert want["off_tile"] == len(info["over"]) and want["cuts"] == 0
            if fmt == K.LTSV:
                assert (c["rounds"], c["direct"]) == (want["rounds"], want["off_tile"])
            else:
                assert (c["rounds"], c["slow"], c["bound_violations"]) == (want["rounds"], want["off_tile"], 0)


@pytest.mark.parametrize("fmt", [K.R5, K.LTSV, K.GELF])
def test_stale_odd_granule(emu, native, oracle, fmt):
    """Second rounds whose byte count is 16 mod 32: the classifier's odd granule holds delimiters of the first round."""
    data, offs, tile = K.stale_granule(fmt, seed=200 + fmt)
    assert K.stale_rounds(offs, tile) == 32
    run(emu, native, oracle, fmt, data, offs, tile)


def test_r5_rounds_at_the_maximum_tile(emu, native, oracle):
    """A batch whose mean clamps pick_tile at the RFC5424 maximum: CTA spans beyond it are cut into rounds at the
    largest tile, and only the lines over 65535 bytes go wide."""
    lines = K.r5_max_tile(seed=310)
    data, offs = K.pack(lines)
    tile = K.batch_tile(K.R5, offs)
    assert tile == K.H100_MAX_TILE5 and int(offs[64] - offs[0]) > tile
    c = run(emu, native, oracle, K.R5, data, offs, tile)
    assert c["wide_lines"] == K.r5_long_wide(lines) and len(c["wide_lines"]) == 4


@pytest.mark.parametrize("eol", [None, b"\n", b"\r\n"])
def test_r5_sixteen_bit_lines(emu, native, oracle, eol):
    """RFC5424 lines of 65534 / 65535 / 65536 bytes (without the terminator) with the SD pair and the message at the far
    end, under a tile that holds all of them: exactly the lines over 65535 bytes go wide."""
    lines, tile = K.r5_sixteen_bit(seed=300)
    if eol is None:
        data, offs = K.pack(lines)
        assert K.batch_tile(K.R5, offs) == tile
        c = run(emu, native, oracle, K.R5, data, offs, tile)
    else:
        data, offs = K.pack([l + eol for l in lines])
        buf, o, c = emu.decode_dump(native, data, offs, tile_bytes=tile, strip_eol=True)
        d0, o0 = K.pack(lines)
        same((buf, o), oracle.decode_dump(K.R5, d0, o0, None, nthreads=8), d0, o0)
    want = K.r5_long_wide(lines)
    assert len(want) == 4 and c["wide_lines"] == want


def test_ltsv_slots_and_direct_next(emu, native, oracle):
    """CTA part totals of 1535 / 1536 / 1537 (+ 64), first lines with more parts than slots (direct_next) and repeated
    `time` parts: the round, cut and direct counts of the restated round loop, exactly."""
    data, offs, info = K.ltsv_slots(seed=400)
    tile = info["tile"]
    assert K.batch_tile(K.LTSV, offs) == tile
    lines = K.lines_of(data, offs)
    rep = repeated_time(lines)
    want = K.slot_rounds(offs, tile, K.ltsv_parts(lines), K.LTSV_SLOTS, True, rep)
    assert want["direct_next"] == 6 and want["cuts"] >= 3 + 6 and want["in_round_direct"] == len(rep) > 0
    c = run(emu, native, oracle, K.LTSV, data, offs, tile)
    assert c["rounds"] == want["rounds"]
    assert c["direct"] == want["off_tile"] + want["in_round_direct"]


def test_ltsv_sixteen_bit_spans(emu, native, oracle):
    data, offs, tile = K.ltsv_sixteen_bit(seed=500)
    assert K.batch_tile(K.LTSV, offs) == tile == 65024
    want = K.slot_rounds(offs, tile, K.ltsv_parts(K.lines_of(data, offs)), K.LTSV_SLOTS, True)
    assert want["off_tile"] == 2 + 2  # the two 65025-byte spans and the two 65535-byte values
    c = run(emu, native, oracle, K.LTSV, data, offs, tile)
    assert (c["rounds"], c["direct"]) == (want["rounds"], want["off_tile"])


@pytest.mark.parametrize("label", [s[0] for s in K.ltsv_schemas()])
def test_ltsv_schema_placement(emu, native, oracle, label):
    """Schemas on both sides of the shared-memory staging limits (64 keys, 1024 name bytes, 64 suffix bytes), keys that
    pass the length and first-byte filters without being schema keys, the empty key, typed values of every type."""
    _, schema, suffixes = next(s for s in K.ltsv_schemas() if s[0] == label)
    data, offs = K.pack(K.ltsv_schema_lines(schema, suffixes, seed=600))
    c = run(emu, native, oracle, K.LTSV, data, offs, K.batch_tile(K.LTSV, offs), cfg=oracle.LtsvConfig(schema, suffixes),
            schema=schema, suffixes=suffixes)
    assert c["schema_staged"] == (not label.endswith(("65", "1025")))


def test_gelf_slots_members_and_numbers(emu, native, oracle):
    """CTA member totals of 1023 / 1024 / 1025, lines of 23 / 24 / 25 members, a round of 1024 members that are mostly
    numbers of more than 6 bytes, and a round of 1024 numbers (both ends of the number list meet): rounds, cuts and the
    slow path of the restated round loop, exactly."""
    data, offs, info = K.gelf_slots(seed=700)
    tile = info["tile"]
    assert K.batch_tile(K.GELF, offs) == tile
    members = K.gelf_members(K.lines_of(data, offs))
    over = sum(m > K.GELF_LOCAL_MEMBERS for m in members)
    want = K.slot_rounds(offs, tile, [m if m <= K.GELF_LOCAL_MEMBERS else 0 for m in members], K.GELF_SLOTS, False)
    assert over > 0 and want["cuts"] >= 1
    c = run(emu, native, oracle, K.GELF, data, offs, tile)
    assert (c["rounds"], c["slow"], c["bound_violations"]) == (want["rounds"], want["off_tile"] + over, 0)


@pytest.mark.parametrize("fmt", [K.LTSV, K.GELF, K.R3164])
def test_one_odd_line_at_every_lane(emu, native, oracle, fmt):
    data, offs = K.lane_mix(fmt, seed=800 + fmt)
    tile = K.batch_tile(fmt, offs)
    lines = K.lines_of(data, offs)
    if fmt == K.R3164:
        c = run(emu, native, oracle, fmt, data, offs, tile, arena_cap=256)
        assert (c["from_tile"], c["from_global"]) == K.r3164_tile_split(offs, tile)
        assert c["from_global"] > 0 and c["redo"] >= 1  # the small arena overflows: regrow and redo, as the C ABI does
        # the 32-threads-per-warp build on the first warp of each pair (the odd line at every lane, ~0.1 s per warp)
        d1, o1 = K.pack([l for w in range(0, len(lines) // 32, 2) for l in lines[32 * w:32 * w + 32]])
        c = run(emu, native, oracle, fmt, d1, o1, K.batch_tile(fmt, o1), warp=True)
        assert c["vote_mismatches"] == 0 and c["votes"] > 0
    elif fmt == K.LTSV:
        rep = repeated_time(lines)
        want = K.slot_rounds(offs, tile, K.ltsv_parts(lines), K.LTSV_SLOTS, True, rep)
        assert want["direct_next"] == 48 and want["in_round_direct"] == 48
        c = run(emu, native, oracle, fmt, data, offs, tile)
        assert (c["rounds"], c["direct"]) == (want["rounds"], want["off_tile"] + want["in_round_direct"])
    else:
        c = run(emu, native, oracle, fmt, data, offs, tile)
        assert c["slow"] >= 3 * 48 and c["bound_violations"] == 0
