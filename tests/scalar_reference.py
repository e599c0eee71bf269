"""Plain-Python reference of greatest, least, nvl2, months_between, date_trunc, make_date, hex, chr, factorial and the local-time
lookups months_between needs.

Integers are Python ints, utf8 / binary values bytes, NULL None.  Time zones come from Python's `zoneinfo`, a reader of the tz
database independent of the engine's own (tzdb.cc).  Only plain Python is used -- no engine, no numpy, no Arrow.

Semantics (Spark's, except where DESIGN.md section 4 records a deviation):
  * greatest / least: NULL arguments skipped, NULL only when all are; the VM's comparison order (floats by IEEE total order,
    bytes unsigned, shorter prefix first); the earlier argument wins a tie
  * nvl2(a, b, c): b when a is not NULL, else c
  * months_between (spark_dates.rs:104-198,403-458): both instants as UTC milliseconds (arrow's cast to Timestamp(ms): a finer
    unit divides toward zero), local dates in the zone (UTC when it is None); the same day of month, or both on the last day of
    their month, gives whole months; otherwise the seconds from each date's local midnight (integer division toward zero) over
    31 days are added; roundOff rounds to 8 digits as floor(x * 1e8 + 0.5) / 1e8
  * date_trunc(level, v): v in its unit truncated toward -inf as a UTC wall clock, converted to the result unit as arrow's cast
    does (a coarser unit divides toward zero); NULL when the level is unknown or the result leaves int64
  * make_date(y, m, d): the day number of a valid proleptic Gregorian date that fits int32, else NULL
  * hex: of an integer the upper-case digits of its 64-bit two's complement without leading zeros, of bytes two per byte
  * chr(n): "" for n < 0, else code point n & 0xFF in UTF-8
  * factorial(n): n! for 0 <= n <= 20, else NULL
"""
from __future__ import annotations

import datetime as dt
import math
import struct
from zoneinfo import ZoneInfo

UTC = dt.timezone.utc
EPOCH = dt.datetime(1970, 1, 1, tzinfo=UTC)
UNIT_PER_S = {"s": 1, "ms": 1000, "us": 10**6, "ns": 10**9}


# ------------------------------------------------------------------------------------------------ greatest / least
def total_f64(x: float) -> int:
    b = struct.unpack("<q", struct.pack("<d", x))[0]
    return b ^ 0x7FFFFFFFFFFFFFFF if b < 0 else b


def total_f32(x: float) -> int:
    b = struct.unpack("<i", struct.pack("<f", x))[0]
    return b ^ 0x7FFFFFFF if b < 0 else b


def order_key(v, kind: str):
    """the VM's comparison order of a value of kind 'int' (ints, dates, timestamps, bool, decimal unscaled), 'f32', 'f64', 'bytes'"""
    if kind == "f64":
        return total_f64(v)
    if kind == "f32":
        return total_f32(v)
    return v


def greatest(vals: list, kind: str, least: bool = False):
    best = None
    for v in vals:
        if v is None:
            continue
        if best is None:
            best = v
            continue
        a, b = order_key(best, kind), order_key(v, kind)
        if (b < a) if least else (b > a):
            best = v
    return best


def nvl2(a, b, c):
    return b if a is not None else c


# ------------------------------------------------------------------------------------------------ dates
def to_ms(v: int, unit: str) -> int:
    """arrow's cast of a timestamp in `unit` (or 'date32' days) to Timestamp(ms)"""
    if unit == "date32":
        return v * 86_400_000
    if unit == "s":
        return v * 1000
    f = UNIT_PER_S[unit] // 1000 if unit != "ms" else 1
    q = abs(v) // f
    return q if v >= 0 else -q


def days_in_month(y: int, m: int) -> int:
    if m == 2:
        return 29 if (y % 4 == 0 and y % 100 != 0) or y % 400 == 0 else 28
    return 30 if m in (4, 6, 9, 11) else 31


def local_date(ms: int, zone: ZoneInfo | None) -> dt.date:
    t = EPOCH + dt.timedelta(milliseconds=ms)
    return (t.astimezone(zone) if zone else t).date()


def start_of_local_day_ms(d: dt.date, zone: ZoneInfo | None) -> int | None:
    """spark_dates.rs:112-139: the earliest instant whose local time is midnight of `d`; in a gap the first minute after it that
    exists"""
    base = dt.datetime(d.year, d.month, d.day)
    if zone is None:
        return (base.replace(tzinfo=UTC) - EPOCH) // dt.timedelta(milliseconds=1)
    for minute in range(0, 24 * 60 + 1):
        local = base + dt.timedelta(minutes=minute)
        hits = []
        for fold in (0, 1):
            u = local.replace(tzinfo=zone, fold=fold).astimezone(UTC)
            if u.astimezone(zone).replace(tzinfo=None) == local:
                hits.append((u - EPOCH) // dt.timedelta(milliseconds=1))
        if hits:
            return min(hits)
    return None


def months_between(ms1, ms2, round_off, zone_name: str | None):
    if ms1 is None or ms2 is None or round_off is None:
        return None
    try:
        zone = ZoneInfo(zone_name) if zone_name else None
    except Exception:   # an unknown zone means UTC (spark_dates.rs:97-102)
        zone = None
    d1, d2 = local_date(ms1, zone), local_date(ms2, zone)
    month_diff = float((d1.year * 12 + d1.month) - (d2.year * 12 + d2.month))
    if d1.day == d2.day or (d1.day == days_in_month(d1.year, d1.month) and d2.day == days_in_month(d2.year, d2.month)):
        return month_diff
    s1, s2 = start_of_local_day_ms(d1, zone), start_of_local_day_ms(d2, zone)
    if s1 is None or s2 is None:
        return None
    sec1, sec2 = int((ms1 - s1) / 1000), int((ms2 - s2) / 1000)   # toward zero; exact for |x| < 2^53
    secs = (d1.day - d2.day) * 86_400 + sec1 - sec2
    r = month_diff + secs / 2_678_400.0
    return math.floor(r * 1e8 + 0.5) / 1e8 if round_off else r


LEVELS = {"YEAR": "year", "YYYY": "year", "YY": "year", "QUARTER": "quarter", "MONTH": "month", "MON": "month", "MM": "month",
          "WEEK": "week", "DAY": "day", "DD": "day", "HOUR": "hour", "MINUTE": "minute", "SECOND": "second",
          "MILLISECOND": "millisecond", "MICROSECOND": "microsecond"}
STEP_NS = {"microsecond": 10**3, "millisecond": 10**6, "second": 10**9, "minute": 60 * 10**9, "hour": 3600 * 10**9, "day": 86400 * 10**9}
UNIT_NS = {"s": 10**9, "ms": 10**6, "us": 10**3, "ns": 1}
I64_MIN, I64_MAX = -(2**63), 2**63 - 1


def date_trunc(fmt, v, unit: str, out_unit: str | None = None):
    out_unit = out_unit or unit
    if v is None or fmt is None or fmt.upper() not in LEVELS:
        return None
    level = LEVELS[fmt.upper()]
    per_day = 86400 * 10**9 // UNIT_NS[unit]
    if level in STEP_NS:
        step = max(1, STEP_NS[level] // UNIT_NS[unit])
        r = v - v % step   # Python's % floors
    else:
        d = v // per_day
        if level == "week":   # Monday; day 0 is a Thursday
            t = d - (d + 3) % 7
        else:
            y, m = _civil(d)
            m = 1 if level == "year" else (m - 1) // 3 * 3 + 1 if level == "quarter" else m
            t = _days_from_civil(y, m, 1)
        r = t * per_day
    if not I64_MIN <= r <= I64_MAX:
        return None
    fo, fi = UNIT_NS[out_unit], UNIT_NS[unit]
    if fo < fi:
        r *= fi // fo
        return r if I64_MIN <= r <= I64_MAX else None
    q = abs(r) // (fo // fi)
    return q if r >= 0 else -q


def _days_from_civil(y: int, m: int, d: int) -> int:   # proleptic Gregorian, any year (Hinnant)
    y -= m <= 2
    era = y // 400
    yoe = y - era * 400
    doy = (153 * (m + (-3 if m > 2 else 9)) + 2) // 5 + d - 1
    doe = yoe * 365 + yoe // 4 - yoe // 100 + doy
    return era * 146097 + doe - 719468


def _civil(days: int) -> tuple[int, int]:
    z = days + 719468
    era = z // 146097
    doe = z - era * 146097
    yoe = (doe - doe // 1460 + doe // 36524 - doe // 146096) // 365
    doy = doe - (365 * yoe + yoe // 4 - yoe // 100)
    mp = (5 * doy + 2) // 153
    m = mp + 3 if mp < 10 else mp - 9
    return yoe + era * 400 + (m <= 2), m


def make_date(y, m, d):
    if y is None or m is None or d is None:
        return None
    if not (1 <= m <= 12 and 1 <= d <= days_in_month(y, m)):
        return None
    z = _days_from_civil(y, m, d)
    return z if -(2**31) <= z < 2**31 else None


# ------------------------------------------------------------------------------------------------ numbers and strings
def factorial(n):
    return None if n is None or not 0 <= n <= 20 else math.factorial(n)


def hex_int(v):
    return None if v is None else format(v & 0xFFFFFFFFFFFFFFFF, "X").encode()


def hex_bytes(b):
    return None if b is None else b.hex().upper().encode()


def chr_(n):
    if n is None:
        return None
    return b"" if n < 0 else chr(n & 0xFF).encode()
