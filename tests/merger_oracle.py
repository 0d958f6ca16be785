"""The reference's Mergers (src/flowgger/merger/*.rs), restated for the tests of the fused encoder's output.framing.
The Output hands every encoded record to its merger before it writes it (output/file_output.rs:209-210,
tls_output.rs:109-110, debug_output.rs:28-29), and a record the decoder rejected is never sent."""
from __future__ import annotations

NONE, LINE, NUL, SYSLEN = 0, 1, 2, 3  # fg_out_framing


def line_merger(record: bytes) -> bytes:
    """line_merger.rs:14: the record, then "\\n"."""
    return record + b"\n"


def nul_merger(record: bytes) -> bytes:
    """nul_merger.rs:14: the record, then "\\0"."""
    return record + b"\0"


def syslen_merger(record: bytes) -> bytes:
    """syslen_merger.rs:15-28: the record gets its "\\n" first, then the decimal of the new length and a space go in
    front of it (so the number counts the "\\n")."""
    framed = record + b"\n"
    return str(len(framed)).encode() + b" " + framed


MERGERS = {NONE: lambda r: r, LINE: line_merger, NUL: nul_merger, SYSLEN: syslen_merger}


def output_stream(records: list[bytes], ok: list[bool], framing: int) -> bytes:
    """What one Output writes for a batch: the merger over the Ok records, in input order."""
    m = MERGERS[framing]
    return b"".join(m(r) for r, good in zip(records, ok) if good)
