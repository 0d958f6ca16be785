"""Every decoder's timestamp against exact integer arithmetic, over the whole calendar.

The reference recipe is `i128 as f64 / 1e9` on the signed nanosecond count of the instant.  Python restates it with no
code in common with the kernels or the oracle: integers are exact, `float(int)` rounds once to nearest-even and `/` is
IEEE division.  The calendar comes from `datetime.date.toordinal` and the local-time rule of RFC3164 zones from
`zoneinfo` (fold=0).

The inputs aim where the arithmetic can go wrong: the calendar's edges (year 0000, negative years, the 100- and 400-year
leap rules, :60, offset hours 24-25, more than nine fraction digits), nanosecond counts that lie on or one unit beside a
rounding tie of the int -> f64 conversion (the sticky-bit branch for |N| >= 2^64), instants within a second of the epoch
(the JSON writer's exponent form) and both sides of every zone transition from 1901 to 2400.

The unmarked tests feed a sub-sample through the CPU emulation of the device logic (tests/emu) and through the oracle;
the `gpu` tests feed every set through the C ABI on the device.
"""
from __future__ import annotations

import datetime
import functools
import random
import re
import sys
from pathlib import Path

import numpy as np
import pytest

R5, LT, R3 = 0, 1, 3
FORMAT_NAMES = {R5: "RFC5424", LT: "LTSV", R3: "RFC3164"}
NS = 1_000_000_000
EPOCH_ORDINAL = datetime.date(1970, 1, 1).toordinal()
ERA_DAYS = 146097                       # days in 400 Gregorian years
MAX_ORDINAL = datetime.date(9999, 12, 31).toordinal()
MONTHS = ["Jan", "Feb", "Mar", "Apr", "May", "Jun", "Jul", "Aug", "Sep", "Oct", "Nov", "Dec"]
ERR_R5 = "Unable to parse the date from RFC3339 to Unix time in RFC5424 decoder"
ERR_LT = "Unable to parse the English to Unix timestamp in LTSV decoder"


# ---- the reference ---------------------------------------------------------------------------------------------------
def _era_shift(y: int) -> int:
    """k such that y + 400 k lies in 1..9999 (datetime's range); the calendar repeats every 400 years"""
    if y < 1:
        return (400 - y) // 400
    if y > 9999:
        return -((y - 9999 + 399) // 400)
    return 0


def is_leap(y: int) -> bool:
    return y % 4 == 0 and (y % 100 != 0 or y % 400 == 0)


def days_in_month(y: int, m: int) -> int:
    return 29 if m == 2 and is_leap(y) else [31, 28, 31, 30, 31, 30, 31, 31, 30, 31, 30, 31][m - 1]


def days_from_civil(y: int, m: int, d: int) -> int:
    """days from 1970-01-01 to y-m-d of the proleptic Gregorian calendar"""
    k = _era_shift(y)
    return datetime.date(y + 400 * k, m, d).toordinal() - ERA_DAYS * k - EPOCH_ORDINAL


def civil_from_days(n: int) -> tuple[int, int, int]:
    o = n + EPOCH_ORDINAL
    k = 0
    while o + ERA_DAYS * k < 1:
        k += 1
    while o + ERA_DAYS * k > MAX_ORDINAL:
        k -= 1
    d = datetime.date.fromordinal(o + ERA_DAYS * k)
    return d.year - 400 * k, d.month, d.day


def expected_ts(n: int) -> float:
    return float(n) / 1e9


def _nanos(frac: str | None) -> int:
    return int((frac or "")[:9].ljust(9, "0"))       # the first nine digits count, later ones are dropped


_RFC3339 = re.compile(r"(\d{4})-(\d{2})-(\d{2})[Tt](\d{2}):(\d{2}):(\d{2})(?:\.(\d+))?(?:[Zz]|([+-])(\d{2}):(\d{2}))", re.ASCII)


def accept_rfc3339(s: str) -> int | None:
    """RFC5424 timestamp / LTSV `time:` in RFC3339: the nanosecond count, or None when rejected"""
    m = _RFC3339.fullmatch(s)
    if not m:
        return None
    y, mo, d, h, mi, sec = (int(m[i]) for i in range(1, 7))
    nanos = _nanos(m[7])
    off = 0
    if m[8]:
        oh, om = int(m[9]), int(m[10])
        if oh > 25 or om > 59:
            return None
        off = (oh * 3600 + om * 60) * (-1 if m[8] == "-" else 1)
    if not (1 <= mo <= 12 and 1 <= d <= days_in_month(y, mo)) or h > 23 or mi > 59 or sec > 60:
        return None
    leap = sec == 60
    if leap:                                           # the leap-second stand-in names :59.999999999
        sec, nanos = 59, NS - 1
    utc = days_from_civil(y, mo, d) * 86400 + h * 3600 + mi * 60 + sec - off
    if leap:                                           # ... and only at the last instant of a month, in UTC
        day, sod = divmod(utc, 86400)
        uy, um, ud = civil_from_days(day)
        if sod != 86399 or ud != days_in_month(uy, um):
            return None
    return utc * NS + nanos


_ENGLISH = re.compile(r"(\d{1,2})/(" + "|".join(MONTHS) + r")/([+-]?\d{4}):(\d{2}):(\d{2}):(\d{2})(?:\.(\d+))? ([+-])(\d{2})(\d{2})",
                      re.ASCII)


def accept_english(s: str) -> int | None:
    """LTSV `time:` as "[day]/[Mon]/[year]:[hour]:[minute]:[second](.[subsecond]) [±HHMM]" (ltsv_decoder.rs:239-247)"""
    m = _ENGLISH.fullmatch(s)
    if not m:
        return None
    d, mo, y = int(m[1]), MONTHS.index(m[2]) + 1, int(m[3])
    h, mi, sec = int(m[4]), int(m[5]), int(m[6])
    oh, om = int(m[9]), int(m[10])
    if d == 0 or d > days_in_month(y, mo) or h > 23 or mi > 59 or sec > 59 or oh > 25 or om > 59:
        return None
    off = (oh * 3600 + om * 60) * (-1 if m[8] == "-" else 1)
    return (days_from_civil(y, mo, d) * 86400 + h * 3600 + mi * 60 + sec - off) * NS + _nanos(m[7])


@functools.lru_cache(maxsize=None)
def _zone(name: str):
    from zoneinfo import ZoneInfo
    return ZoneInfo(name)


def zone_offset(name: str, local: int) -> int:
    """UTC offset in force at the local second `local` of zone `name`, fold=0"""
    wall = datetime.datetime(1970, 1, 1) + datetime.timedelta(seconds=local)
    return int(wall.replace(tzinfo=_zone(name)).utcoffset().total_seconds())


FIXED_ZONES = {"UTC": 0, "Etc/GMT+12": -12 * 3600, "Etc/GMT-14": 14 * 3600}   # no transitions: valid in every year


def accept_rfc3164(line: str, year: int, zones) -> int | None:
    """The stamp of "[[±]YYYY ]Mon D HH:MM:SS [zone ]h m": without a year the context's year applies (only when it has
    four digits); a known zone identifier after the time gives the offset of that local time."""
    tok = line.split(" ")
    if tok[0] in MONTHS:
        if not 1000 <= year <= 9999:
            return None
        i = 0
    else:
        if not re.fullmatch(r"[+-]?\d{4}", tok[0], re.ASCII):
            return None
        year, i = int(tok[0]), 1
    if tok[i] not in MONTHS or not re.fullmatch(r"\d{1,2}", tok[i + 1], re.ASCII):
        return None
    mo, d = MONTHS.index(tok[i]) + 1, int(tok[i + 1])
    t = re.fullmatch(r"(\d{2}):(\d{2}):(\d{2})", tok[i + 2], re.ASCII)
    if not t or d == 0 or d > days_in_month(year, mo):
        return None
    h, mi, sec = int(t[1]), int(t[2]), int(t[3])
    if h > 23 or mi > 59 or sec > 59:
        return None
    local = days_from_civil(year, mo, d) * 86400 + h * 3600 + mi * 60 + sec
    z = tok[i + 3]
    if z in FIXED_ZONES:
        local -= FIXED_ZONES[z]
    elif z in zones:
        local -= zone_offset(z, local)
    return local * NS


# ---- rendering -------------------------------------------------------------------------------------------------------
def _wall(n: int, off: int):
    secs, nanos = divmod(n, NS)
    day, sod = divmod(secs + off, 86400)
    y, mo, d = civil_from_days(day)
    return y, mo, d, sod // 3600, sod // 60 % 60, sod % 60, nanos


def _off3339(off: int, big_z: bool = True) -> str:
    if off is None:
        return "Z" if big_z else "z"
    a = abs(off)
    return f"{'-' if off < 0 else '+'}{a // 3600:02d}:{a // 60 % 60:02d}"


def render_rfc3339(n: int, off: int | None = None, lower: bool = False) -> str | None:
    """the instant n written with `off` seconds of offset (None: Z) and 9 fraction digits; None outside years 0..9999"""
    y, mo, d, h, mi, s, ns = _wall(n, off or 0)
    if not 0 <= y <= 9999:
        return None
    return f"{y:04d}-{mo:02d}-{d:02d}{'t' if lower else 'T'}{h:02d}:{mi:02d}:{s:02d}.{ns:09d}{_off3339(off, not lower)}"


def render_english(n: int, off: int = 0) -> str | None:
    y, mo, d, h, mi, s, ns = _wall(n, off)
    if not -9999 <= y <= 9999:
        return None
    a = abs(off)
    return (f"{d}/{MONTHS[mo - 1]}/{'-' if y < 0 else ''}{abs(y):04d}:{h:02d}:{mi:02d}:{s:02d}.{ns:09d} "
            f"{'-' if off < 0 else '+'}{a // 3600:02d}{a // 60 % 60:02d}")


def _digits(rng: random.Random, k: int) -> str:
    return f"{rng.getrandbits(48) % 10**12:012d}"[:k]


# ---- input sets ------------------------------------------------------------------------------------------------------
YEARS = [0, 1, 3, 4, 99, 100, 399, 400, 1000, 1384, 1385, 1582, 1600, 1677, 1678, 1899, 1900, 1969, 1970, 1971, 2000, 2038,
         2100, 2261, 2262, 2263, 2400, 2553, 2554, 2555, 9998, 9999]
DAYS = [0, 1, 28, 29, 30, 31, 32]
TIMES = ["00:00:00", "23:59:59", "24:00:00", "23:60:00", "23:59:60"]
OFF_MINUTES = [0, 1, 30, 59, 60]
OFFSETS_3339 = ["Z", "z", "+00:00", "-00:00"] + [f"{s}{h:02d}:{m:02d}" for s in "+-" for h in range(27) for m in OFF_MINUTES]
OFFSETS_ENGLISH = [f"{s}{h:02d}{m:02d}" for s in "+-" for h in range(27) for m in OFF_MINUTES]
NEAR_EPOCH = [1, 9, 10, 999, 1000, 999_999, 1_000_000, 1_000_001, 123_456_789, NS - 1]
N_MIN_3339 = days_from_civil(0, 1, 1) * 86400 * NS
N_MAX_3339 = (days_from_civil(9999, 12, 31) + 1) * 86400 * NS - 1
N_MIN_ENGLISH = days_from_civil(-9999, 1, 1) * 86400 * NS


def tie_counts(rng: random.Random, n_min: int, n_max: int) -> list[int]:
    """N = m·ulp + ulp/2 + δ around 2^k (ulp = 2^(k-52), δ ∈ {-1, 0, +1}), m even and odd, both signs, for every k the
    range [n_min, n_max] reaches; the extreme mantissas 2^52 and 2^53 - 1 (rounding up into the next binade) included"""
    out = []
    for k in range(53, 72):
        ulp = 1 << (k - 52)
        for sign in (1, -1):
            lim = n_max if sign > 0 else -n_min
            m_hi = min((1 << 53) - 1, (lim - ulp // 2 - 1) // ulp)
            if m_hi < 1 << 52:
                continue
            ms = {1 << 52, m_hi}
            for parity in (0, 1):
                for _ in range(3):
                    m = rng.randrange(1 << 52, m_hi + 1)
                    m += (m & 1) != parity
                    ms.add(m if m <= m_hi else m - 2)
            out += [sign * (m * ulp + ulp // 2 + delta) for m in sorted(ms) for delta in (-1, 0, 1)]
    return out


class Lines:
    """lines of one format, with the model's nanosecond count (None: rejected) and a kind tag per line"""

    def __init__(self):
        self.lines: list[bytes] = []
        self.n: list[int | None] = []
        self.kind: list[str] = []

    def add(self, line: str, n: int | None, kind: str):
        self.lines.append(line.encode())
        self.n.append(n)
        self.kind.append(kind)

    def __len__(self):
        return len(self.lines)

    def pack(self, idx=None):
        import pyoracle
        return pyoracle.pack(self.lines if idx is None else [self.lines[i] for i in idx])

    @functools.cached_property
    def accepted(self) -> np.ndarray:
        return np.array([n is not None for n in self.n], dtype=bool)

    @functools.cached_property
    def bits(self) -> np.ndarray:
        return np.array([expected_ts(n) if n is not None else 0.0 for n in self.n], dtype=np.float64).view(np.uint64)

    def sample(self, rng: random.Random, keep_random: int) -> list[int]:
        """every grid, tie and near-epoch line, and `keep_random` of the others"""
        fixed = [i for i, k in enumerate(self.kind) if not k.startswith(("random", "zone"))]
        rest = [i for i, k in enumerate(self.kind) if k.startswith(("random", "zone"))]
        return fixed + sorted(rng.sample(rest, min(keep_random, len(rest))))


def rfc3339_stamps(n_random: int) -> list[tuple[str, str, int | None]]:
    """(stamp, kind, N the generator meant or None when it did not aim at a valid stamp)"""
    rng = random.Random(3339)
    out = []
    for y in YEARS:                                    # the calendar grid: year x month x day x time, all of it
        for mo in range(1, 13):
            for d in DAYS:
                for t in TIMES:
                    fl = rng.randrange(13)
                    frac = "." + _digits(rng, fl) if fl else ""
                    out.append((f"{y:04d}-{mo:02d}-{d:02d}{'t' if rng.random() < 0.1 else 'T'}{t}{frac}{rng.choice(OFFSETS_3339)}",
                                "grid", None))
    for n in tie_counts(rng, N_MIN_3339, N_MAX_3339):
        off = rng.choice([60, 7 * 3600 + 30 * 60, 23 * 3600 + 59 * 60]) * (-1 if n > 0 else 1)
        out += [(render_rfc3339(n), "tie:fast", n), (render_rfc3339(n, off), "tie:fast", n), (render_rfc3339(n, lower=True), "tie:slow", n),
                (render_rfc3339(n, 25 * 3600 * (-1 if n > 0 else 1)), "tie:slow", n)]
    for n in NEAR_EPOCH + [-v for v in NEAR_EPOCH]:
        z = render_rfc3339(n)
        out += [(z, "near:fast", n), (render_rfc3339(n, -5 * 3600), "near:fast", n), (render_rfc3339(n, 24 * 3600 + 60), "near:slow", n),
                (render_rfc3339(n, lower=True), "near:slow", n), (z[:-1] + "999Z", "near:slow", n)]   # digits past the ninth
    lo, hi = N_MIN_3339 // NS, N_MAX_3339 // NS
    for _ in range(n_random):                          # random instants over 0000-01-01 .. 9999-12-31
        utc = rng.randrange(lo, hi + 1)
        fl = rng.randrange(13)
        frac = _digits(rng, fl)
        slow = rng.random() < 0.1
        if rng.random() < 0.15:
            off = None
        else:
            off = rng.randrange(-23 * 3600 - 59 * 60, 24 * 3600, 60)
            if slow and rng.random() < 0.5:
                off = rng.choice([1, -1]) * rng.randrange(24 * 3600, 25 * 3600 + 59 * 60 + 1, 60)
        n = utc * NS + _nanos(frac)
        y, mo, d, h, mi, s, _ = _wall(n, off or 0)
        if not 0 <= y <= 9999:
            off = None
            y, mo, d, h, mi, s, _ = _wall(n, 0)
        tz = _off3339(off, not slow)
        out.append((f"{y:04d}-{mo:02d}-{d:02d}{'t' if slow else 'T'}{h:02d}:{mi:02d}:{s:02d}{'.' + frac if fl else ''}{tz}",
                    "random:slow" if slow else "random", n))
    return out


def english_stamps(n_random: int) -> list[tuple[str, str, int | None]]:
    rng = random.Random(1414)
    out = []
    for y in sorted(set(YEARS + [-y for y in YEARS])):
        for mo in range(1, 13):
            for d in DAYS:
                for t in TIMES:
                    fl = rng.randrange(13)
                    ds = str(d) if d >= 10 or rng.random() < 0.7 else f"{d:02d}"
                    ys = ("-" if y < 0 else rng.choice(["", "", "+"])) + f"{abs(y):04d}"
                    out.append((f"{ds}/{MONTHS[mo - 1]}/{ys}:{t}{'.' + _digits(rng, fl) if fl else ''} {rng.choice(OFFSETS_ENGLISH)}",
                                "grid", None))
    out.append(("5/Aug/-0000:00:00:00 +0000", "grid", None))
    for n in tie_counts(rng, N_MIN_ENGLISH, N_MAX_3339):
        off = rng.choice([60, 7 * 3600 + 1800, 25 * 3600 + 59 * 60]) * (-1 if n > 0 else 1)
        out += [(render_english(n), "tie", n), (render_english(n, off), "tie", n)]
    for n in NEAR_EPOCH + [-v for v in NEAR_EPOCH]:
        out += [(render_english(n), "near", n), (render_english(n, 3600), "near", n)]
    lo, hi = N_MIN_ENGLISH // NS, N_MAX_3339 // NS
    for _ in range(n_random):
        utc = rng.randrange(lo, hi + 1)
        n = utc * NS + (rng.randrange(NS) if rng.random() < 0.5 else 0)
        s = render_english(n, rng.randrange(-25 * 3600 - 59 * 60, 26 * 3600, 60))
        if s is None:
            s = render_english(n)
        if n % NS == 0 and rng.random() < 0.5:
            s = s.replace(".000000000", "")            # the form without .subsecond
        out.append((s, "random", n))
    return out


@functools.lru_cache(maxsize=None)
def rfc5424_set(n_random: int) -> Lines:
    L = Lines()
    for s, kind, want in rfc3339_stamps(n_random):
        n = accept_rfc3339(s)
        assert want is None or n == want, (s, n, want)          # the renderer and the acceptor agree
        L.add(f"<13>1 {s} h a p m - x", n, kind)
    return L


@functools.lru_cache(maxsize=None)
def ltsv_set(n_random: int) -> Lines:
    L = Lines()
    for s, kind, want in rfc3339_stamps(n_random):
        n = accept_rfc3339(s)
        assert want is None or n == want, (s, n, want)
        L.add(f"time:{s}\thost:h", n, kind)
    for s, kind, want in english_stamps(n_random // 4):
        n = accept_english(s)
        assert want is None or n == want, (s, n, want)
        L.add(f"time:[{s}]\thost:h", n, kind)
    return L


CONTEXT_YEARS = (1000, 2000, 2024, 2026, 2100, 9999)


@functools.lru_cache(maxsize=None)
def rfc3164_set(n_random: int) -> Lines:
    """lines that carry their year: the grid (zone-less, or with a zone of one fixed offset) and random instants"""
    rng = random.Random(3164)
    L = Lines()
    zones = [None, None] + sorted(FIXED_ZONES)
    for y in sorted(set(YEARS + [-y for y in YEARS])):
        for mo in range(1, 13):
            for d in DAYS:
                for t in TIMES:
                    ys = ("-" if y < 0 else rng.choice(["", "", "+"])) + f"{abs(y):04d}"
                    ds = str(d) if d >= 10 or rng.random() < 0.7 else f"{d:02d}"
                    z = rng.choice(zones)
                    line = f"{ys} {MONTHS[mo - 1]} {ds} {t} {z + ' ' if z else ''}h m"
                    L.add(line, accept_rfc3164(line, 0, ()), "grid")
    lo, hi = days_from_civil(-9999, 1, 1) * 86400, days_from_civil(9999, 12, 31) * 86400 + 86399
    for _ in range(n_random):
        local = rng.randrange(lo, hi + 1)
        y, mo, d, h, mi, s, _ = _wall(local * NS, 0)
        z = rng.choice(zones)
        ys = f"{'-' if y < 0 else ''}{abs(y):04d}"
        line = f"{ys} {MONTHS[mo - 1]} {d} {h:02d}:{mi:02d}:{s:02d} {z + ' ' if z else ''}h m"
        n = accept_rfc3164(line, 0, ())
        assert n == (local - FIXED_ZONES.get(z, 0)) * NS, line
        L.add(line, n, "random")
    return L


@functools.lru_cache(maxsize=None)
def rfc3164_yearless_set(year: int) -> Lines:
    """month x day x time without a year: the context's year applies (Feb 29 only in a leap year)"""
    rng = random.Random(year)
    L = Lines()
    for mo in range(1, 13):
        for d in DAYS:
            for t in TIMES:
                ds = str(d) if d >= 10 or rng.random() < 0.7 else f"{d:02d}"
                z = rng.choice([None, "UTC", "Etc/GMT-14"])
                line = f"{MONTHS[mo - 1]} {ds} {t} {z + ' ' if z else ''}h m"
                L.add(line, accept_rfc3164(line, year, ()), "grid")
    return L


@functools.lru_cache(maxsize=None)
def zone_set() -> Lines:
    """For every zone both the default zone table and zoneinfo know, every transition from 1901 to 2400: the local times
    transition + offset before + d and transition + offset after + d (d = -1, 0, +1), and the middle of each span.
    Zones are interleaved, so that neighbouring lines (the lanes of one warp) search different zones."""
    import tzread
    from zoneinfo import available_timezones
    known = available_timezones()
    tables = tzread.load_zones()
    lo = days_from_civil(1901, 1, 2) * 86400
    hi = days_from_civil(2399, 12, 30) * 86400
    per_zone = []
    for name in sorted(set(tables) & known):
        tr, of = tables[name]
        probes = []
        for k, t in enumerate(tr):
            if not lo <= t <= hi:
                continue
            for o in (of[k], of[k + 1]):
                probes += [t + o + d for d in (-1, 0, 1)]
            if k + 1 < len(tr) and tr[k + 1] <= hi:
                probes.append((t + tr[k + 1]) // 2 + of[k + 1])
        if probes:
            per_zone.append((name, probes))
    L = Lines()
    for j in range(max(len(p) for _, p in per_zone)):
        for name, probes in per_zone:
            if j < len(probes):
                local = probes[j]
                y, mo, d, h, mi, s, _ = _wall(local * NS, 0)
                L.add(f"{y:04d} {MONTHS[mo - 1]} {d} {h:02d}:{mi:02d}:{s:02d} {name} h m", (local - zone_offset(name, local)) * NS,
                      "zone")
    return L


# ---- comparisons -----------------------------------------------------------------------------------------------------
def dump_fields(buf: bytes, offs: np.ndarray) -> tuple[np.ndarray, np.ndarray, list]:
    """per line of a canonical dump: accepted?, ts bits, error text (None when accepted)"""
    n = len(offs) - 1
    ok = np.zeros(n, dtype=bool)
    bits = np.zeros(n, dtype=np.uint64)
    err = [None] * n
    for i in range(n):
        d = buf[offs[i]:offs[i + 1]]
        if d.startswith(b"R:ts="):
            ok[i] = True
            bits[i] = int(d[5:21], 16)
        else:
            assert d.startswith(b"E:"), d
            err[i] = d[2:].split(b";out=")[0].decode()
    return ok, bits, err


def check_model(who: str, L: Lines, idx, ok: np.ndarray, bits: np.ndarray):
    """a line is accepted exactly when the model accepts it, and then carries exactly float(N) / 1e9"""
    idx = np.asarray(idx)
    want_ok, want_bits = L.accepted[idx], L.bits[idx]
    bad = np.nonzero((ok != want_ok) | (want_ok & (bits != want_bits)))[0]
    if len(bad):
        msg = []
        for j in bad[:8]:
            i = int(idx[j])
            want = "rejected" if L.n[i] is None else f"{int(want_bits[j]):016x} (N={L.n[i]})"
            got = f"{int(bits[j]):016x}" if ok[j] else "rejected"
            msg.append(f"  {L.lines[i]!r} [{L.kind[i]}]: model {want}, got {got}")
        raise AssertionError(f"{who}: {len(bad)} of {len(idx)} lines differ from the model\n" + "\n".join(msg))


_PLAIN = re.compile(r"-?(0|[1-9][0-9]*)\.[0-9]+")
_EXPONENT = re.compile(r"-?[1-9](\.[0-9]+)?e-?[1-9][0-9]*")


def check_json_number(text: str, v: float) -> bool:
    """serde's shape of an f64, round-tripping to exactly v; True when written in exponent form"""
    assert np.float64(float(text)).view(np.uint64) == np.float64(v).view(np.uint64), (text, v)
    if v == 0.0:
        assert text == ("-0.0" if np.signbit(v) else "0.0"), (text, v)
        return False
    if 1e-6 <= abs(v) < 1e21:
        assert _PLAIN.fullmatch(text), (text, v)
        return False
    assert _EXPONENT.fullmatch(text), (text, v)
    return True


def coverage(L: Lines, idx=None) -> dict[str, int]:
    idx = range(len(L)) if idx is None else idx
    c = {"lines": 0, "accepted": 0, "|N|>=2^64": 0, "tie": 0}
    for i in idx:
        c["lines"] += 1
        c["tie"] += L.kind[i].startswith("tie")
        if L.n[i] is not None:
            c["accepted"] += 1
            c["|N|>=2^64"] += abs(L.n[i]) >= 1 << 64
    return c


# ---- the model itself ------------------------------------------------------------------------------------------------
def test_model_rules():
    """the reference restates the rules it is meant to, on hand-picked stamps"""
    assert days_from_civil(1970, 1, 1) == 0 and days_from_civil(2000, 3, 1) == 11017
    assert days_from_civil(0, 1, 1) == -719528 and days_from_civil(-1, 12, 31) == -719529
    assert days_from_civil(-400, 1, 1) == -719528 - ERA_DAYS
    for n in (-3_652_059 - 719_528, -719_529, -1, 0, 59, 2_932_896):
        assert days_from_civil(*civil_from_days(n)) == n
    assert is_leap(0) and is_leap(-4) and is_leap(2000) and not is_leap(1900) and not is_leap(-100) and is_leap(-400)
    a = accept_rfc3339
    assert a("1970-01-01T00:00:00Z") == 0 and a("1970-01-01t00:00:00.000000001z") == 1
    assert a("1969-12-31T23:59:59.999999999999Z") == -1                       # the tenth digit is dropped, not rounded
    assert a("2016-12-31T23:59:60Z") == a("2016-12-31T23:59:59.999999999Z") == a("2016-12-31T18:59:60.5-05:00")
    assert a("2016-12-31T22:59:60Z") is None and a("2016-06-30T23:59:60+00:00") is not None and a("2016-06-29T23:59:60Z") is None
    assert a("2015-08-05T15:53:45+25:59") is not None and a("2015-08-05T15:53:45+26:00") is None
    assert a("2015-08-05T15:53:45.Z") is None and a("2015-08-05T15:53:45") is None and a("2015-08-05T24:00:00Z") is None
    assert a("2015-02-29T00:00:00Z") is None and a("2000-02-29T00:00:00Z") and a("1900-02-29T00:00:00Z") is None
    assert a("0000-02-29T00:00:00Z") is not None and a("٢٠١٥-08-05T15:53:45Z") is None
    e = accept_english
    assert e("10/Oct/2000:13:55:36 -0700") == 971211336 * NS
    assert e("5/Aug/-0044:15:53:45 -0000") is not None and e("0/Aug/2015:15:53:45 +0130") is None
    assert e("5/aug/2015:15:53:45 +0130") is None and e("5/Aug/2015:15:53:60 +0000") is None
    assert e("5/Aug/2015:15:53:45 0130") is None and e("5/Aug/2015:15:53:45.123456789123 +0000") == e("5/Aug/2015:15:53:45.123456789 +0000")
    r = accept_rfc3164
    assert r("2020 Aug 6 11:15:24 h m", 0, ()) == 1596712524 * NS
    assert r("Feb 29 00:00:00 h m", 2024, ()) is not None and r("Feb 29 00:00:00 h m", 2026, ()) is None
    assert r("Feb 29 00:00:00 h m", 999, ()) is None and r("-0001 Feb 29 00:00:00 h m", 0, ()) is None
    assert r("2021 Mar 14 02:30:00 America/New_York h m", 0, {"America/New_York"}) == 1615707000 * NS
    assert r("2021 Nov 7 01:30:00 America/New_York h m", 0, {"America/New_York"}) == 1636263000 * NS
    assert r("2020 Aug 6 11:15:24 Etc/GMT+12 h m", 0, ()) == (1596712524 + 12 * 3600) * NS
    # the renderers write what the acceptors read back
    rng = random.Random(1)
    for n in tie_counts(rng, N_MIN_3339, N_MAX_3339)[::7] + [N_MIN_3339, N_MAX_3339]:
        assert accept_rfc3339(render_rfc3339(n)) == n
    assert accept_english(render_english(N_MIN_ENGLISH)) == N_MIN_ENGLISH


def test_input_sets_cover_every_axis():
    """every value of every grid axis appears; ties reach 2^68, past the 2^64 of the conversion's second branch"""
    stamps = [s for s, k, _ in rfc3339_stamps(0) if k == "grid"]
    for off in OFFSETS_3339:
        assert any(s.endswith(off) for s in stamps), off
    for fl in range(13):
        pat = re.compile(r".{19}" + (r"\.\d{%d}" % fl if fl else "") + r"([Zz]|[+-]\d\d:\d\d)")
        assert any(pat.fullmatch(s) for s in stamps), fl
    eng = [s for s, k, _ in english_stamps(0) if k == "grid"]
    for off in OFFSETS_ENGLISH:
        assert any(s.endswith(" " + off) for s in eng), off
    assert any(s.split("/")[2].startswith("-9999") for s in eng)
    ties = tie_counts(random.Random(0), N_MIN_ENGLISH, N_MAX_3339)
    ks = {abs(n).bit_length() - 1 for n in ties}
    assert ks == set(range(53, 69)), sorted(ks)
    assert min(ties) < -(1 << 68) and max(ties) > 1 << 67


# ---- CPU: the emulation of the device logic and the oracle, against the model ---------------------------------------
CPU_RANDOM = 60_000


@pytest.fixture(scope="module")
def emu():
    sys.path.insert(0, str(Path(__file__).resolve().parent / "emu"))
    import emu as E
    E.build()
    return E


def test_rfc5424_emulation_and_oracle(emu, native, oracle):
    L = rfc5424_set(CPU_RANDOM)
    data, offs = L.pack()
    for who, (buf, bo) in (("emulation", emu.decode_dump(native, data, offs)[:2]), ("oracle", oracle.decode_dump(R5, data, offs))):
        ok, bits, err = dump_fields(buf, bo)
        check_model(f"RFC5424 {who}", L, range(len(L)), ok, bits)
        assert {e for e in err if e is not None} == {ERR_R5}
    c = coverage(L)
    print(f"RFC5424 CPU: {c}")
    assert c["|N|>=2^64"] > 0 and c["tie"] > 0


def test_ltsv_emulation_and_oracle(emu, native, oracle):
    L = ltsv_set(4 * CPU_RANDOM)
    idx = L.sample(random.Random(5), 70_000)
    data, offs = L.pack(idx)
    for who, (buf, bo) in (("emulation", emu.ltsv_decode_dump(native, data, offs)[:2]), ("oracle", oracle.decode_dump(LT, data, offs))):
        ok, bits, err = dump_fields(buf, bo)
        check_model(f"LTSV {who}", L, idx, ok, bits)
        assert {e for e in err if e is not None} == {ERR_LT}
    c = coverage(L, idx)
    print(f"LTSV CPU: {c}")
    assert c["|N|>=2^64"] > 0 and c["tie"] > 0


def test_rfc3164_emulation_and_oracle(emu, native, oracle):
    parts = [(rfc3164_set(CPU_RANDOM // 2), 2026, None)]
    parts += [(rfc3164_yearless_set(y), y, None) for y in CONTEXT_YEARS]
    Z = zone_set()
    parts.append((Z, 2026, sorted(random.Random(7).sample(range(len(Z)), min(len(Z), 60_000)))))
    for L, year, idx in parts:
        idx = range(len(L)) if idx is None else idx
        data, offs = L.pack(idx)
        cfg = oracle.Rfc3164Config(year)
        # r3164_parse_lockstep is what the kernel runs; r3164_parse_line restates it one line at a time
        for who, (buf, bo) in (("lock-step emulation", emu.r3164_decode_dump(native, data, offs, year)[:2]),
                               ("per-line emulation", emu.r3164_decode_dump(native, data, offs, year, lockstep=False)[:2]),
                               ("oracle", oracle.decode_dump(R3, data, offs, cfg))):
            ok, bits, _ = dump_fields(buf, bo)
            check_model(f"RFC3164 {who} (year {year})", L, idx, ok, bits)
    print(f"RFC3164 CPU: {coverage(parts[0][0])}, zone probes {len(parts[-1][2])} of {len(Z)}")
    assert coverage(parts[0][0])["|N|>=2^64"] > 0


def test_json_writer_emulation_and_oracle(emu, oracle):
    """the device's JSON number writer (emulated) and the oracle's print the model's value of every accepted RFC5424
    line of the grid, tie and near-epoch sets in serde's shape, round-tripping exactly"""
    import ctypes as C
    f = emu.lib().emu_json_f64
    f.argtypes = [C.c_double, C.c_char_p]
    buf = C.create_string_buffer(40)
    L = rfc5424_set(0)
    values = {expected_ts(n) for n in L.n if n is not None}
    exp_form = 0
    for v in sorted(values):
        k = f(v, buf)
        dev = buf.raw[:k].decode()
        ref = oracle.format_f64(v)
        exp_form += check_json_number(dev, v)
        check_json_number(ref, v)
        assert dev == ref, (v, dev, ref)
    print(f"JSON writer CPU: {len(values)} values, {exp_form} in exponent form")
    assert exp_form > 0


# ---- GPU: every set through the C ABI --------------------------------------------------------------------------------
GPU_RANDOM = 1_000_000


def _decode(native, fmt: int, L: Lines, year: int = 0):
    data, offs = L.pack()
    dec = native.BatchDecoder(fmt, max_batch_bytes=int(offs[-1]) + (1 << 20), max_batch_lines=len(L), rfc3164_year=year)
    try:
        res = dec.decode(data, offs)
        status = np.array(res.status)
        ts = np.array(res.ts)
    finally:
        dec.close()
    return data, offs, status, ts


def _check_device(native, oracle, fmt, L: Lines, data, offs, status, ts, cfg=None):
    check_model(f"{FORMAT_NAMES[fmt]} on the GPU", L, range(len(L)), status == 0, np.where(status == 0, ts.view(np.uint64), 0))
    obuf, ooffs = oracle.decode_dump(fmt, data, offs, cfg)
    _, _, oerr = dump_fields(obuf, ooffs)
    for i in np.nonzero(status)[0]:
        assert native.error_string(fmt, int(status[i])) == oerr[i], (L.lines[i], int(status[i]), oerr[i])


def _same_instant_same_bits(L: Lines, ts: np.ndarray):
    """every instant written in the fast-path shape and in a slow-path shape decodes to the same bits"""
    fast, slow = {}, {}
    for i, (k, n) in enumerate(zip(L.kind, L.n)):
        if n is not None and k.endswith(("fast", "slow")):
            (fast if k.endswith("fast") else slow).setdefault(n, set()).add(int(ts.view(np.uint64)[i]))
    both = fast.keys() & slow.keys()
    assert len(both) > 100
    for n in both:
        assert len(fast[n] | slow[n]) == 1, n


@pytest.mark.gpu
def test_rfc5424_on_gpu(native, oracle):
    L = rfc5424_set(GPU_RANDOM)
    data, offs, status, ts = _decode(native, native.FMT_RFC5424, L)
    _check_device(native, oracle, native.FMT_RFC5424, L, data, offs, status, ts)
    _same_instant_same_bits(L, ts)
    c = coverage(L)
    print(f"RFC5424 GPU: {c}")
    assert c["|N|>=2^64"] > 0 and c["tie"] > 0


@pytest.mark.gpu
def test_ltsv_on_gpu(native, oracle):
    L = ltsv_set(GPU_RANDOM)
    data, offs, status, ts = _decode(native, native.FMT_LTSV, L)
    _check_device(native, oracle, native.FMT_LTSV, L, data, offs, status, ts)
    _same_instant_same_bits(L, ts)
    c = coverage(L)
    print(f"LTSV GPU: {c}")
    assert c["|N|>=2^64"] > 0 and c["tie"] > 0


@pytest.mark.gpu
def test_rfc3164_calendar_on_gpu(native, oracle):
    L = rfc3164_set(GPU_RANDOM // 4)
    data, offs, status, ts = _decode(native, native.FMT_RFC3164, L, year=2026)
    _check_device(native, oracle, native.FMT_RFC3164, L, data, offs, status, ts, oracle.Rfc3164Config(2026))
    for year in CONTEXT_YEARS:
        Y = rfc3164_yearless_set(year)
        data, offs, status, ts = _decode(native, native.FMT_RFC3164, Y, year=year)
        _check_device(native, oracle, native.FMT_RFC3164, Y, data, offs, status, ts, oracle.Rfc3164Config(year))
        feb29 = [i for i, l in enumerate(Y.lines) if l.startswith(b"Feb 29 00:00:00")]
        assert (status[feb29] == 0).all() == is_leap(year)
    print(f"RFC3164 GPU: {coverage(L)}")


@pytest.mark.gpu
def test_rfc3164_zone_transitions_on_gpu(native):
    Z = zone_set()
    _, _, status, ts = _decode(native, native.FMT_RFC3164, Z, year=2026)
    check_model("rfc3164 zone transitions on the GPU", Z, range(len(Z)), status == 0, np.where(status == 0, ts.view(np.uint64), 0))
    zones = {l.split(b" ")[4] for l in Z.lines}
    print(f"RFC3164 GPU: {len(Z)} zone-transition probes in {len(zones)} zones")
    assert len(Z) > 100_000 and len(zones) > 300


@pytest.mark.gpu
def test_gelf_encoder_timestamps_on_gpu(native, oracle):
    import json
    L = rfc5424_set(0)
    data, offs = L.pack()
    dec = native.BatchDecoder(native.FMT_RFC5424, max_batch_bytes=int(offs[-1]) + (1 << 20), max_batch_lines=len(L))
    try:
        buf, joffs, status, _ = dec.decode_encode_gelf(data, offs)
    finally:
        dec.close()
    assert ((status == 0) == L.accepted).all()
    pat = re.compile(rb'"timestamp":([^,}]+)')
    exp_form = 0
    for i in np.nonzero(L.accepted)[0]:
        rec = buf[joffs[i]:joffs[i + 1]]
        json.loads(rec)
        (text,) = pat.findall(rec)
        v = expected_ts(L.n[i])
        exp_form += check_json_number(text.decode(), v)
        assert text.decode() == oracle.format_f64(v), (L.lines[i], text, oracle.format_f64(v))
    print(f"GELF encoder GPU: {int(L.accepted.sum())} records, {exp_form} timestamps in exponent form")
    assert exp_form > 0
