"""PassthroughEncoder::encode (src/flowgger/encoder/passthrough_encoder.rs:22-46) restated over the oracle's decoded
Records, for the tests of the fused passthrough encoder.  The Records come from the oracle's canonical dumps
(oracle.decode_dump, read by ltsv_oracle.parse_dump), so Record.full_msg is the oracle decoder's; the encoder is
restated here: the header (output.syslog_prepend_timestamp, already formatted) followed by full_msg, or the error
NO_RAW for a Record without full_msg (and then no header either)."""
from __future__ import annotations

from ltsv_oracle import parse_dump

NO_RAW = "Cannot output empty raw message"  # passthrough_encoder.rs:44
FG_EP_NO_RAW = 128  # its status (fg_status.h): above every decoder status


def encode(full: bytes | None, header: bytes = b"") -> bytes | None:
    """passthrough_encoder.rs:22-46 over Record.full_msg: header + full_msg, or None for Err(NO_RAW)"""
    return None if full is None else header + full


def decode_records(oracle, fmt: int, data, offsets, cfg=None, nthreads: int = 8) -> list:
    """the oracle's Record of every line (None for a line the decoder rejects)"""
    buf, offs = oracle.decode_dump(fmt, data, offsets, cfg=cfg, nthreads=nthreads)
    return [parse_dump(buf[offs[i]:offs[i + 1]], 0.0) for i in range(len(offs) - 1)]


def decode_encode_passthrough(oracle, fmt: int, data, offsets, header: bytes = b"", cfg=None,
                              nthreads: int = 8) -> tuple[list[bytes], list[bool]]:
    """decode + PassthroughEncoder::encode per line: (one record per line, b"" for a line the decoder or the encoder
    rejects; per line, whether the encoder rejected it with NO_RAW)"""
    out, no_raw = [], []
    for rec in decode_records(oracle, fmt, data, offsets, cfg, nthreads):
        r = None if rec is None else encode(rec["full"], header)
        out.append(b"" if r is None else r)
        no_raw.append(rec is not None and r is None)
    return out, no_raw
