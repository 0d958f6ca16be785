"""oracle/pyrfc3164.py — TEST INFRASTRUCTURE: a second, independent restatement of RFC3164Decoder::decode
(flowgger src/flowgger/decoder/rfc3164_decoder.rs:31-213) in plain Python.

It shares no code with oracle/rfc3164.cpp or with the product: tokens come from a regular expression over Rust's
White_Space set, dates from `datetime`, zones from the standard library's `zoneinfo` (fold = 0) instead of the TZif readers
of oracle/tzread.py and flowgger_b200/csrc/fg_tz.cu, timestamps from Python's correctly rounded int -> float conversion.
tests/test_oracle_golden.py::test_rfc3164_three_way compares it with the C++ oracle line by line; anything it cannot
express (years outside 1..9999, which `datetime` does not have) returns UNSUPPORTED and is skipped there.
"""
from __future__ import annotations

import re
from datetime import datetime, timezone
from zoneinfo import ZoneInfo, available_timezones

UNSUPPORTED = object()
PANIC = "(the reference panics here: index out of bounds, rfc3164_decoder.rs:64)"

# char::is_whitespace
_WS = "\t\n\x0b\x0c\r \x85\xa0  -     　"
_TOKEN = re.compile(f"[^{_WS}]+")
_TRAIL = re.compile(f"[{_WS}]+\\Z")
_MONTHS = {m: i + 1 for i, m in enumerate("Jan Feb Mar Apr May Jun Jul Aug Sep Oct Nov Dec".split())}
_YEAR = re.compile(r"[+-]?[0-9]{4}\Z")
_DAY = re.compile(r"[0-9]{1,2}\Z")
_TIME = re.compile(r"([0-9]{2}):([0-9]{2}):([0-9]{2})\Z")
_ZONES = None


def _zones():
    global _ZONES
    if _ZONES is None:
        _ZONES = available_timezones() - {"localtime", "posixrules"}
    return _ZONES


def _u8(s: str):
    """u8::from_str"""
    if s.startswith("+"):
        s = s[1:]
    if not s or not s.isascii() or not s.isdigit():
        return None
    v = int(s)
    return v if v <= 255 else None


def _primitive(year_tok: str, mon: str, day: str, tm: str):
    """PrimitiveDateTime::parse over "[year] [month repr:short] [day padding:none] [hour]:[minute]:[second]" -> naive
    datetime, None (parse error) or UNSUPPORTED."""
    if not (_YEAR.match(year_tok) and year_tok.isascii()):
        return None
    if mon not in _MONTHS or not (_DAY.match(day) and day.isascii()):
        return None
    m = _TIME.match(tm)
    if not m or not tm.isascii():
        return None
    y, d = int(year_tok), int(day)
    hh, mm, ss = (int(x) for x in m.groups())
    if d == 0 or hh > 23 or mm > 59 or ss > 59:
        return None
    if y < 1 or y > 9999:
        # `time` accepts years -9999..9999; datetime does not: validate the day by hand, then give up on the value
        leap = (y % 4 == 0 and y % 100 != 0) or y % 400 == 0
        dim = [31, 29 if leap else 28, 31, 30, 31, 30, 31, 31, 30, 31, 30, 31][_MONTHS[mon] - 1]
        return UNSUPPORTED if d <= dim else None
    try:
        return datetime(y, _MONTHS[mon], d, hh, mm, ss)
    except ValueError:
        return None


def _parse_date(tokens: list[str], has_year: bool, year: int):
    """parse_date (:163-213) -> (ts, tokens consumed) | error string | UNSUPPORTED"""
    if has_year:
        if len(tokens) < 4:
            return "Unable to parse RFC3164 date with year"
        dt, idx = _primitive(tokens[0], tokens[1], tokens[2], tokens[3]), 4
    else:
        dt, idx = _primitive(str(year), tokens[0], tokens[1], tokens[2]), 3
    if dt is None:
        return "Unable to parse the date in RFC3164 decoder"
    if dt is UNSUPPORTED:
        return UNSUPPORTED
    if len(tokens) > idx and tokens[idx] in _zones():
        aware = dt.replace(tzinfo=ZoneInfo(tokens[idx]), fold=0)
        idx += 1
    else:
        aware = dt.replace(tzinfo=timezone.utc)
    delta = aware - datetime(1970, 1, 1, tzinfo=timezone.utc)
    secs = delta.days * 86400 + delta.seconds
    return float(secs * 1_000_000_000) / 1e9, idx  # unix_timestamp_nanos() as f64 / 1e9 (utils/mod.rs:24-35)


def _parse_date_token(tokens: list[str], year: int):
    if len(tokens) < 3:
        return "Invalid time format"
    r = _parse_date(tokens, False, year)
    if r is UNSUPPORTED or isinstance(r, tuple):
        return r
    return _parse_date(tokens, True, year)


def decode(line: str, year: int):
    """-> dict(ts, hostname, facility, severity, msg, full_msg) | error string | UNSUPPORTED"""
    fac = sev = None
    msg = line
    if line.startswith("<"):
        k = line.find(">")
        if k < 0:
            return "Malformed RFC3164 event: Invalid priority"
        pri = _u8(line[:k + 1].lstrip("<").rstrip(">"))
        if pri is None:
            return "Invalid priority"
        fac, sev, msg = pri >> 3, pri & 7, line[k + 1:]
    full = _TRAIL.sub("", line)
    tok = _TOKEN.findall(msg)
    if len(tok) > 3:
        r = _parse_date_token(tok, year)
        if r is UNSUPPORTED:
            return UNSUPPORTED
        if isinstance(r, tuple):
            ts, idx = r
            if idx >= len(tok):
                return PANIC
            return dict(ts=ts, hostname=tok[idx], facility=fac, severity=sev, msg=" ".join(tok[idx + 1:]), full_msg=full)
    parts = msg.split(": ")
    if len(parts) <= 2:
        return "Malformed RFC3164 event: Invalid timestamp or hostname"
    r = _parse_date_token(_TOKEN.findall(parts[1]), year)
    if r is UNSUPPORTED or isinstance(r, str):
        return r
    return dict(ts=r[0], hostname=parts[0], facility=fac, severity=sev, msg=": ".join(parts[2:]), full_msg=full)


def dump(res) -> bytes:
    """the canonical parity dump of oracle.cpp::dump for an RFC3164 result"""
    import struct
    if isinstance(res, str):
        return b"E:" + res.encode() + b";out=0"

    def s(x: str) -> bytes:
        b = x.encode()
        return str(len(b)).encode() + b":" + b

    def o(v):
        return b"~" if v is None else str(v).encode()
    return (b"R:ts=" + struct.pack(">d", res["ts"]).hex().encode() + b";fac=" + o(res["facility"]) + b";sev=" + o(res["severity"]) +
            b";host=" + s(res["hostname"]) + b";app=~;proc=~;msgid=~;msg=" + s(res["msg"]) + b";full=" + s(res["full_msg"]) +
            b";sd=~;out=0")
