"""oracle/pysplit.py — TEST INFRASTRUCTURE: CPU restatement of the framing LineSplitter::run performs before decode
(flowgger src/flowgger/splitter/line_splitter.rs:17-25): `BufRead::lines` (split at b'\\n', drop it and ONE
preceding b'\\r'; an unterminated last line is still yielded; an empty stream yields nothing) and the UTF-8 check of
`String` (invalid => the line is skipped with "Invalid UTF-8 input")."""
from __future__ import annotations

import numpy as np


def split_lines(stream: bytes) -> tuple[np.ndarray, list[bytes], list[bool]]:
    """Returns (line start offsets int32[n+1] incl. terminators, stripped lines, utf8-valid flags)."""
    a = np.frombuffer(stream, dtype=np.uint8)
    nl = np.flatnonzero(a == 10)
    starts = [0] + [int(p) + 1 for p in nl]
    if len(stream) > 0 and stream[-1] != 10:
        starts.append(len(stream))
    if len(stream) == 0:
        return np.zeros(1, np.int32), [], []
    offs = np.asarray(starts, dtype=np.int32)
    lines, valid = [], []
    for i in range(len(offs) - 1):
        l = stream[offs[i]:offs[i + 1]]
        if l.endswith(b"\n"):
            l = l[:-1]
            if l.endswith(b"\r"):
                l = l[:-1]
        lines.append(l)
        try:
            l.decode("utf-8")
            valid.append(True)
        except UnicodeDecodeError:
            valid.append(False)
    return offs, lines, valid


def split_nul(stream: bytes) -> tuple[np.ndarray, list[bytes], list[bool]]:
    """NulSplitter::run (flowgger src/flowgger/splitter/nul_splitter.rs:18-40): `BufRead::split(0)` — records end at
    a NUL byte, which is dropped; nothing else is stripped; an unterminated last record is still yielded; invalid UTF-8 =>
    "Invalid UTF-8 input" and the record is skipped.  Same return shape as split_lines."""
    if len(stream) == 0:
        return np.zeros(1, np.int32), [], []
    a = np.frombuffer(stream, dtype=np.uint8)
    z = np.flatnonzero(a == 0)
    starts = [0] + [int(p) + 1 for p in z]
    if stream[-1] != 0:
        starts.append(len(stream))
    offs = np.asarray(starts, dtype=np.int32)
    lines, valid = [], []
    for i in range(len(offs) - 1):
        l = stream[offs[i]:offs[i + 1]]
        if l.endswith(b"\0"):
            l = l[:-1]
        lines.append(l)
        try:
            l.decode("utf-8")
            valid.append(True)
        except UnicodeDecodeError:
            valid.append(False)
    return offs, lines, valid
